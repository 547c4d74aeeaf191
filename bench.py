#!/usr/bin/env python
"""bench.py — BGZF inflate (+ CRAM rANS-Nx16 decode) throughput on H100, beside the reference's
CPU path on the same machine.  See DESIGN.md §Measurement.

One "step" = one pass of the BGZF inflate hot path over the whole synthetic 150 bp BAM
(BASELINE.json configs[1]: 10 GB uncompressed, zlib level 6, one warp per 64 KiB block).
  value      uncompressed GB/s, kernel with inputs resident in HBM (CUDA events)
  e2e        same metric through the C-ABI host entry point (hgpu_bgzf_inflate_file_host) with
             pinned HOST buffers: H2D of the compressed file + kernel + D2H of the output, timed
  roofline   (C+U) algorithmic bytes / kernel time against MEASURED_PEAKS.json hbm_gbs
  cpu_baseline  the unmodified reference (oracle/_ref/libhts_ref.so: bgzf_read + bgzf_mt thread
             pool) on the host cores, on a bounded sample of the same file
  extra.rans CRAM 3.1 rANS-Nx16 decode (BASELINE.json configs[2]) measured after the timed steps

--dump-outputs DIR writes what the last timed step computed, for comparing two builds output for output:
  block_len.npy, block_status.npy   per BGZF block: inflated length and status (float64)
  inflated_sample.npy               DUMP_SAMPLE bytes of the inflated stream (float32) at positions drawn
                                    with numpy default_rng(0).integers(0, uncompressed bytes), sorted
The corpus is generated from fixed seeds, so the same arguments give the same inputs on every run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--gb", type=float, default=10.0, help="uncompressed BAM gigabytes per GPU (10 = BASELINE configs[1])")
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--quals", default="novaseq")
    ap.add_argument("--rans-slices", type=int, default=-2, help="CRAM slices for the rANS leg (0 = skip)")
    ap.add_argument("--tok3-blocks", type=int, default=9472, help="read-name blocks for the tok3 leg (0 = skip)")
    ap.add_argument("--cram-tiles", type=int, default=120, help="CRAM record-decode leg: the reference-written 100k-read file tiled this many times (0 = skip)")
    ap.add_argument("--cpu-sample-gb", type=float, default=4.0)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's outputs as .npy files to DIR")
    return ap.parse_args()


DUMP_SAMPLE = 12 << 20                  # 48 MB of float32: the whole dump stays under 64 MB


def dump_outputs(out_dir, torch, d_out, U, d_len, d_st):
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "block_len.npy"), d_len.cpu().numpy().astype(np.float64))
    np.save(os.path.join(out_dir, "block_status.npy"), d_st.cpu().numpy().astype(np.float64))
    pos = np.sort(np.random.default_rng(0).integers(0, U, size=min(U, DUMP_SAMPLE)))
    idx = torch.from_numpy(pos).to(d_out.device)
    np.save(os.path.join(out_dir, "inflated_sample.npy"), d_out[idx].cpu().numpy().astype(np.float32))


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s HBM3)"


class ClockSampler:
    """nvidia-smi clocks/throttle reasons DURING the timed region."""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index = index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except OSError:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            pass
        sm = sorted(int(r[0]) for r in self.rows if r and r[0].isdigit())
        mx = [int(r[1]) for r in self.rows if len(r) > 1 and r[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[k] for r in self.rows if len(r) >= 6 for k in range(4) if r[2 + k].lower().startswith("active")})
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


# --------------------------------------------------------------------------------------------
# reference arm: the unmodified reference built into oracle/_ref (bgzf_read over bgzf_mt)
# --------------------------------------------------------------------------------------------
def ref_lib():
    so = os.path.join(ROOT, "oracle", "_ref", "libhts_ref.so")
    if not os.path.exists(so):
        return None
    r = C.CDLL(so)
    r.hopen.restype = C.c_void_p
    r.hopen.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t]
    r.bgzf_hopen.restype = C.c_void_p
    r.bgzf_hopen.argtypes = [C.c_void_p, C.c_char_p]
    r.bgzf_read.restype = C.c_ssize_t
    r.bgzf_read.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bgzf_mt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.hfile_mem_steal_buffer.restype = C.c_void_p
    r.hfile_mem_steal_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
    return r


def ref_decompress(r, img, threads):
    """bgzip -d equivalent in-process: mem: hFILE -> bgzf_hopen -> bgzf_mt(threads) -> bgzf_read loop.
    img: np.uint8 BGZF file image.  Returns (uncompressed bytes, seconds)."""
    libc = C.CDLL(None)
    libc.malloc.restype = C.c_void_p
    libc.malloc.argtypes = [C.c_size_t]
    mem = libc.malloc(img.size)                       # the mem: backend frees it at close
    C.memmove(mem, img.ctypes.data, img.size)
    t0 = time.perf_counter()
    hf = r.hopen(b"mem:", b"r:", mem, img.size)
    fp = r.bgzf_hopen(hf, b"r")
    if threads > 1:
        r.bgzf_mt(fp, threads, 256)
    buf = (C.c_uint8 * (16 << 20))()
    total = 0
    while True:
        n = r.bgzf_read(fp, buf, len(buf))
        if n <= 0:
            break
        total += n
    r.bgzf_close(fp)
    return total, time.perf_counter() - t0


def cpu_sample(corpus, sample_bytes):
    from tools import synth
    ulen, clen = corpus["ulen"], corpus["clen"]
    cu = np.cumsum(ulen.astype(np.int64))
    nb = int(np.searchsorted(cu, sample_bytes)) + 1
    nb = min(nb, len(ulen))
    cbytes = int(clen[:nb].astype(np.int64).sum())
    img = np.concatenate([corpus["comp"][:cbytes], np.frombuffer(synth.BGZF_EOF, dtype=np.uint8)])
    return img, int(cu[nb - 1]), cbytes, nb


def run_cpu_baseline(corpus, sample_gb, reps=2):
    r = ref_lib()
    cores = len(os.sched_getaffinity(0))
    if r is None:
        return None
    img, ubytes, cbytes, nb = cpu_sample(corpus, sample_gb * 1e9)
    best = None
    for _ in range(reps):
        total, sec = ref_decompress(r, img, cores)
        assert total == ubytes, (total, ubytes)
        best = sec if best is None else min(best, sec)
    return {"value": ubytes / best / 1e9, "unit": "GB/s", "cores": cores, "kind": "reference",
            "sample": "first %d BGZF blocks (%.2f GB uncompressed) of the same file, bgzf_read over bgzf_mt(%d threads), zlib arm, best of %d"
                      % (nb, ubytes / 1e9, cores, reps)}


# --------------------------------------------------------------------------------------------
def make_corpus(args, rank, world=1):
    """Per-GPU corpus of args.gb uncompressed GB.  At N=1 every block is unique.  At N>1 the host
    cores are shared by N generators, so each rank makes gb/N unique GB (own seed) and repeats it N
    times at distinct addresses: per-GPU work stays fixed (weak scaling) and far larger than L2."""
    from tools import synth
    t0 = time.time()
    procs = max(1, len(os.sched_getaffinity(0)) // world)
    corpus = synth.bam_bgzf_corpus(args.gb * 1e9 / world, level=args.level, quals=args.quals, seed=42 + rank, procs=procs)
    if world > 1:
        corpus["comp"] = np.tile(corpus["comp"], world)
        corpus["clen"] = np.tile(corpus["clen"], world)
        corpus["ulen"] = np.tile(corpus["ulen"], world)
        corpus["n_reads"] *= world
    corpus["tile"] = world
    corpus["gen_s"] = time.time() - t0
    return corpus


def rans_legs(args, ctx, torch, dev, world, dist):
    """BASELINE.json configs[2]: CRAM 3.1 rANS-Nx16 decode of 30x-WGS-shaped slices, streams written by the
    UNMODIFIED reference encoder (tools/rans_bench.py), NovaSeq 4-bin and HiSeq ~40-value qualities, every
    block compared on the device with the generator's input; device time, host-buffer (e2e) time and the
    reference decoder on the host cores beside it.  Runs at every N (slices shard without a collective)."""
    import gc
    import htslib_b200 as H
    from tools import rans_bench
    if args.rans_slices == 0:
        return None
    waves = -args.rans_slices if args.rans_slices < 0 else 1
    out = {}
    for alphabet in ("novaseq", "hiseq"):
        # each alphabet on a context of its own, closed afterwards: its device staging (as large as the batch)
        # is released before the next one, so both fit next to the other legs in 80 GB
        gc.collect()
        torch.cuda.empty_cache()
        rctx = H.Context(dev.index)
        try:
            out[alphabet] = rans_bench.run(rctx, torch, dev, peaks(), alphabet=alphabet, waves=waves, reps=5, world=world,
                                           dist=dist, e2e=not args.no_e2e, cpu=(world == 1 and not args.no_cpu_baseline))
        except Exception as ex:                                   # the headline line must still print
            out[alphabet] = {"error": repr(ex)}
        finally:
            rctx.close()
    head = dict(out["novaseq"])
    head["hiseq"] = out["hiseq"]
    head["note"] = ("top level = NovaSeq 4-bin qualities (SURVEY.md 8d first data set); 'hiseq' = the 40-value data set; "
                    "value = uncompressed GB/s over all GPUs, roofline = (C+U)/t per GPU against the measured copy bandwidth")
    return head


def bind_to_gpu_numa(local):
    """Pin this rank's threads (and therefore its first-touch pinned staging) to the NUMA node its GPU
    hangs off: at N>1 the host side of the e2e path is otherwise bound by cross-socket traffic."""
    try:
        import re
        bus = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=pci.bus_id", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=20).stdout.strip().lower()
        if not bus:
            return None
        if len(bus.split(":")[0]) == 8:
            bus = bus[4:]
        node = int(open("/sys/bus/pci/devices/%s/numa_node" % bus).read().strip())
        if node < 0:
            return None
        cpus = open("/sys/devices/system/node/node%d/cpulist" % node).read().strip()
        ids = set()
        for part in cpus.split(","):
            lo, _, hi = part.partition("-")
            ids.update(range(int(lo), int(hi or lo) + 1))
        ids &= os.sched_getaffinity(0)
        if ids:
            os.sched_setaffinity(0, ids)
        return {"numa_node": node, "cpus": len(ids)}
    except Exception:
        return None


def strong_leg(args, ctx, torch, dev, dist, world, rank, corpus, d_in, d_io, d_il, d_out, d_oo, d_cap, d_len, d_st, stream, steps):
    """STRONG split (SURVEY.md 8e): ONE file of args.gb uncompressed GB whose blocks shard across the ranks in
    contiguous ranges (hgpu_shard_range).  The file is the concatenation, in rank order, of the first 1/N of
    every rank's resident corpus (each rank generated its own blocks).  Per step: rank 0 broadcasts the BAM
    header block over NCCL, the ranks all-gather their ranges' uncompressed lengths (-> global output bases),
    each rank inflates its own range; time = max over ranks; no collective on the data path."""
    import htslib_b200 as H
    clen, ulen = corpus["clen"], corpus["ulen"]
    k = len(clen) // world                                  # blocks of this rank's part
    kk = torch.tensor([k], device=dev, dtype=torch.int64)
    dist.all_reduce(kk, op=dist.ReduceOp.MIN)
    k = int(kk.item())
    # the global unit table every rank needs for hgpu_shard_range: the uncompressed length of every block of the file
    mine = torch.from_numpy(ulen[:k].astype(np.int32)).to(dev)
    allu = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allu, mine)
    g_ulen = torch.cat(allu).cpu().numpy().astype(np.uint32)
    first, count, out_base = H.shard_range(g_ulen, world, rank)
    assert count == k and first == rank * k, (first, count, k)
    hdr_txt = ("@HD\tVN:1.6\tSO:coordinate\n" + "".join("@SQ\tSN:chr%d\tLN:%d\n" % (c + 1, 248956422 - c * 5000000) for c in range(24))
               + "@RG\tID:grp1\tSM:synthetic\n").encode()
    hdr = torch.zeros(len(hdr_txt), dtype=torch.uint8, device=dev)
    if rank == 0:
        hdr.copy_(torch.frombuffer(bytearray(hdr_txt), dtype=torch.uint8))
    my_u = torch.tensor([int(ulen[:k].astype(np.int64).sum())], device=dev, dtype=torch.int64)
    lens = [torch.zeros_like(my_u) for _ in range(world)]
    sl = slice(0, k)
    a_io, a_il, a_oo, a_cap = d_io[sl].contiguous(), d_il[sl].contiguous(), d_oo[sl].contiguous(), d_cap[sl].contiguous()
    a_len, a_st = d_len[sl].contiguous(), d_st[sl].contiguous()

    def step():
        dist.broadcast(hdr, src=0)                          # the one collective north_star names: header (and reference) to every rank
        dist.all_gather(lens, my_u)                         # global output bases = prefix sums of these
        ctx.bgzf_inflate_dev(d_in, a_io, a_il, d_out, a_oo, a_cap, a_len, a_st, stream)
    for _ in range(2):
        step()
    torch.cuda.synchronize(); dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    tt = torch.tensor([e0.elapsed_time(e1)], device=dev)
    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms = float(tt.item()) / steps
    dist.barrier()
    assert int(a_st.abs().sum().item()) == 0
    assert bytes(hdr.cpu().numpy().tobytes()) == hdr_txt
    tot = int(sum(int(x.item()) for x in lens))
    assert int(np.cumsum([0] + [int(x.item()) for x in lens])[rank]) == out_base
    return {"scaling": "strong", "value": tot / ms / 1e6, "unit": "GB/s", "ms_per_step": ms, "uncompressed_bytes_total": tot,
            "blocks_per_gpu": k, "collectives_per_step": "NCCL broadcast of the BAM header block (%d B) + all-gather of %d x 8 B range lengths; none on the data path" % (len(hdr_txt), world),
            "shard": "hgpu_shard_range: rank r takes blocks [r*k, (r+1)*k) and writes at the global output base the all-gather gives"}


def run_ours(args):
    import torch
    import htslib_b200 as H
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py needs a GPU (there is no CPU fallback)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    ctx = H.Context(local)
    corpus = make_corpus(args, rank, world)
    numa = bind_to_gpu_numa(local) if world > 1 else None       # after the generators: they want every core
    comp, clen, ulen = corpus["comp"], corpus["clen"], corpus["ulen"]
    nb = len(clen)
    in_off = np.concatenate([[0], np.cumsum(clen.astype(np.int64))[:-1]]).astype(np.uint64)
    out_off = np.concatenate([[0], np.cumsum(ulen.astype(np.int64))[:-1]]).astype(np.uint64)
    U, Cb = int(ulen.astype(np.int64).sum()), int(clen.astype(np.int64).sum())
    t = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32)).to(dev)
    d_in = torch.empty(Cb + 64, dtype=torch.uint8, device=dev)
    d_in[:Cb].copy_(torch.from_numpy(comp.copy()))
    d_out = torch.empty(U + 64, dtype=torch.uint8, device=dev)
    d_io, d_il, d_oo, d_cap = t(in_off), t(clen), t(out_off), t(ulen)
    d_len = torch.zeros(nb, dtype=torch.int32, device=dev)
    d_st = torch.zeros(nb, dtype=torch.int32, device=dev)
    # a real stream: handle 0 (legacy default) would make the library fall back to its own stream,
    # which torch.cuda.Event on the current stream cannot see
    tstream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    torch.cuda.set_stream(tstream)
    stream = tstream.cuda_stream
    assert stream != 0
    L = H.lib()

    def step():
        ctx.bgzf_inflate_dev(d_in, d_io, d_il, d_out, d_oo, d_cap, d_len, d_st, stream)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    # correctness gate before timing: every block OK, lengths right, stream CRCs match the generator
    assert int(d_st.abs().sum().item()) == 0, "inflate reported errors"
    assert bool((d_len.cpu().numpy().astype(np.uint32) == ulen).all())
    import zlib
    # shards were compressed independently; check the first shard's CRC32 end to end
    k_shard = corpus["shard_blocks"][0]
    crc = zlib.crc32(d_out[:int(ulen[:k_shard].astype(np.int64).sum())].cpu().numpy().tobytes())
    assert crc == corpus["shard_crcs"][0], "first shard CRC mismatch"

    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    torch.cuda.synchronize()
    launches0 = L.hgpu_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    launches = L.hgpu_launch_count() - launches0
    ms_total = e0.elapsed_time(e1)
    if world > 1:
        import torch.distributed as dist
        tt = torch.tensor([ms_total], device=dev)
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        ms_total = float(tt.item())
        dist.barrier()
    clocks = sampler.stop() if rank == 0 else None
    ms_step = ms_total / args.steps
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, torch, d_out, U, d_len, d_st)

    # ---- BAM record unpack over the inflated stream, still on the device (configs[3] front half) ----
    bam_extra = None
    if True:                                                     # every rank: its own shard (times = max over ranks below)
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = ctx.bam_unpack_dev(d_out, U, d_oo, True, stream)
            torch.cuda.synchronize()
            first = time.perf_counter() - t0
            n_rec = r["n"]
            bad = int((r["status"] != 0).sum().item())
            written = int(r["data_off"][n_rec].item()) + 2 * int(r["seq_off"][n_rec].item()) + 48 * n_rec
            del r
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            r = ctx.bam_unpack_dev(d_out, U, d_oo, True, stream)
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1)
            hbm, how = peaks()
            bam_extra = {"workload": "record index + layout + unpack (bam1_core_t, data, ASCII SEQ, QUAL+33) of the inflated stream",
                         "records": n_rec, "bad_records": bad, "ms": ms, "includes": "two small D2H syncs for counts/sizes and output allocation",
                         "records_per_s": n_rec / ms * 1e3, "value": U / ms / 1e6, "unit": "GB/s (input stream)",
                         "roofline": {"bound": "hbm", "achieved": (U + written) / ms / 1e6, "peak": hbm, "unit": "GB/s",
                                      "frac": (U + written) / ms / 1e6 / hbm, "traffic": None, "peak_source": how}}
            assert bad == 0 and (world > 1 or n_rec == corpus["n_reads"])
            # ---- BAM -> SAM text (configs[3]): sam_format1 of every record on the device ----
            try:
                text, t_off, t_st = ctx.sam_format_dev(r["core"], r["data"], r["data_off"], n_rec, [b"chr1"], stream)
                torch.cuda.synchronize()
                del text, t_off
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                text, t_off, t_st = ctx.sam_format_dev(r["core"], r["data"], r["data_off"], n_rec, [b"chr1"], stream)
                ev1.record()
                torch.cuda.synchronize()
                sms = ev0.elapsed_time(ev1)
                bam_extra["sam_text"] = {"ms": sms, "text_bytes": int(text.numel()), "text_GBps": int(text.numel()) / sms / 1e6,
                                         "records_per_s": n_rec / sms * 1e3, "flagged_for_host": int((t_st != 0).sum().item()),
                                         "includes": "layout pass, one D2H of the total, output allocation, write pass (hgpu_sam_format_dev twice)"}
                del text, t_off, t_st
            except Exception as ex:
                bam_extra["sam_text"] = {"error": repr(ex)}
            # ---- write half of the BAM round trip (configs[3]): pack (bam_write1) + BGZF compress ----
            try:
                packed, pk_off, pk_st = ctx.bam_pack_dev(r["core"], r["data"], r["data_off"], n_rec, stream)
                torch.cuda.synchronize()
                same = bool(torch.equal(packed, d_out[:U]))
                nblk = (U + 0xff00 - 1) // 0xff00
                pin_off = torch.arange(nblk, dtype=torch.int64, device=dev) * 0xff00
                pin_len = torch.full((nblk,), 0xff00, dtype=torch.int32, device=dev)
                pin_len[-1] = U - (nblk - 1) * 0xff00
                c_out = torch.empty(nblk * 65536 + 64, dtype=torch.uint8, device=dev)
                c_off = torch.arange(nblk, dtype=torch.int64, device=dev) * 65536
                c_len = torch.zeros(nblk, dtype=torch.int32, device=dev); c_st = torch.zeros(nblk, dtype=torch.int32, device=dev)
                def squeeze():
                    H.check(L.hgpu_bgzf_compress_batch_dev(ctx.h, packed.data_ptr(), pin_off.data_ptr(), pin_len.data_ptr(), nblk, 6,
                                                           c_out.data_ptr(), c_off.data_ptr(), c_len.data_ptr(), c_st.data_ptr(), stream), "compress")
                squeeze(); torch.cuda.synchronize()
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(); squeeze(); ev1.record(); torch.cuda.synchronize()
                cms = ev0.elapsed_time(ev1)
                csz = int(c_len.sum().item())
                ev0.record()
                packed2, _, _ = ctx.bam_pack_dev(r["core"], r["data"], r["data_off"], n_rec, stream)
                ev1.record(); torch.cuda.synchronize()
                pms = ev0.elapsed_time(ev1)
                # re-inflate the first 2000 of our own blocks on the device and compare with the stream
                k = min(nblk, 2000)
                chk = torch.zeros(k * 65536, dtype=torch.uint8, device=dev)
                cap = torch.full((k,), 65536, dtype=torch.int32, device=dev)
                ol = torch.zeros(k, dtype=torch.int32, device=dev); st2 = torch.zeros(k, dtype=torch.int32, device=dev)
                ctx.bgzf_inflate_dev(c_out, c_off[:k].contiguous(), c_len[:k].contiguous(), chk, c_off[:k].contiguous(), cap, ol, st2, stream)
                torch.cuda.synchronize()
                ok = int(st2.abs().sum().item()) == 0 and bool((ol == pin_len[:k]).all().item())
                ok = ok and bool(torch.equal(chk.view(k, 65536)[0, :0xff00], packed[:0xff00]))
                bam_extra["write_half"] = {"pack_ms": pms, "pack_GBps": U / pms / 1e6, "pack_reproduces_stream": same,
                                           "deflate_ms": cms, "deflate_GBps": U / cms / 1e6, "deflate_level": ">=1 (LZ77 + dynamic / fixed Huffman, smaller per block)",
                                           "compressed_bytes": csz, "ratio": csz / U, "zlib6_ratio": Cb / U,
                                           "size_vs_zlib6": csz / Cb, "reinflate_check": ok, "errors": int(c_st.abs().sum().item())}
                del packed, packed2, c_out, chk
            except Exception as ex:
                bam_extra["write_half"] = {"error": repr(ex)}
            del r
        except Exception as ex:
            bam_extra = {"error": repr(ex)}

    if world > 1:
        # every rank reaches this all-reduce whatever happened above: times become the max over ranks, rates the aggregate
        v = [0.0, 0.0, 0.0, 0.0, 0.0]
        try:
            if bam_extra and "ms" in bam_extra:
                v = [1.0, bam_extra["ms"], bam_extra.get("sam_text", {}).get("ms", 0.0), bam_extra.get("write_half", {}).get("pack_ms", 0.0),
                     bam_extra.get("write_half", {}).get("deflate_ms", 0.0)]
        except Exception:
            pass
        tt = torch.tensor(v, dtype=torch.float64, device=dev)
        mn = tt.clone()
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        if bam_extra and "ms" in bam_extra and float(mn[0].item()) == 1.0:
            ms_u, ms_s, ms_p, ms_d = (float(x) for x in tt[1:].tolist())
            bam_extra.update({"n_gpus": world, "ms": ms_u, "records_per_s": world * bam_extra["records"] / ms_u * 1e3, "value": world * U / ms_u / 1e6,
                              "unit": "GB/s (input stream, all GPUs)", "aggregation": "every rank unpacks its own inflated shard; time = max over ranks"})
            if ms_s and "ms" in bam_extra.get("sam_text", {}):
                bam_extra["sam_text"].update({"ms": ms_s, "text_GBps": world * bam_extra["sam_text"]["text_bytes"] / ms_s / 1e6,
                                              "records_per_s": world * bam_extra["records"] / ms_s * 1e3})
            if ms_p and "pack_ms" in bam_extra.get("write_half", {}):
                bam_extra["write_half"].update({"pack_ms": ms_p, "pack_GBps": world * U / ms_p / 1e6, "deflate_ms": ms_d, "deflate_GBps": world * U / ms_d / 1e6})
        elif bam_extra is not None and "error" not in bam_extra:
            bam_extra = {"error": "a rank failed this leg"}

    d_out_keep = d_out
    # ---- e2e: host buffers through the C-ABI file entry point ----
    e2e = None
    if not args.no_e2e:
        from tools import synth
        h_file = torch.empty(Cb + len(synth.BGZF_EOF), dtype=torch.uint8).pin_memory()
        h_file[:Cb].copy_(torch.from_numpy(comp.copy()))
        h_file[Cb:].copy_(torch.frombuffer(bytearray(synth.BGZF_EOF), dtype=torch.uint8))
        h_out = torch.empty(U, dtype=torch.uint8).pin_memory()
        fn, on = h_file.numpy(), h_out.numpy()
        rc, n, bad = ctx.bgzf_inflate_file_host(fn, on)           # warm-up (allocates staging)
        assert rc == 0 and n == U, (rc, n, bad, H.last_error())
        assert zlib.crc32(on[:int(ulen[:k_shard].astype(np.int64).sum())].tobytes()) == corpus["shard_crcs"][0]
        reps = max(2, min(args.steps, 5))
        if world > 1:
            dist.barrier()
        t0 = time.perf_counter()
        for _ in range(reps):
            rc, n, bad = ctx.bgzf_inflate_file_host(fn, on)
        torch.cuda.synchronize()
        sec = (time.perf_counter() - t0) / reps
        if world > 1:
            tt = torch.tensor([sec], device=dev)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            sec = float(tt.item())
        e2e = {"value": U * world / sec / 1e9, "unit": "GB/s", "h2d_bytes_per_step": Cb + len(synth.BGZF_EOF) + nb * 24,
               "d2h_bytes_per_step": U + nb * 8, "api": "hgpu_bgzf_inflate_file_host (pinned host buffers, 3-stream chunk pipeline)"}
        del h_file, h_out

    # ---- legs every rank takes part in ----
    strong = None
    if world > 1:
        try:
            strong = strong_leg(args, ctx, torch, dev, dist, world, rank, corpus, d_in, d_io, d_il, d_out_keep, d_oo, d_cap, d_len, d_st, stream, max(2, min(args.steps, 5)))
        except Exception as ex:
            strong = {"error": repr(ex)}
    del d_in, d_out_keep, d_out
    torch.cuda.empty_cache()
    rans = None
    try:
        rans = rans_legs(args, ctx, torch, dev, world, dist)
    except Exception as ex:
        rans = {"error": repr(ex)}
    # ---- CRAM record decode + encode (configs[4] shape), every rank on its own copy of the reference-written file ----
    cram = None
    if args.cram_tiles > 0:
        try:
            sys.path.insert(0, os.path.join(ROOT, "tools"))
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import cram_records_bench
            cram = cram_records_bench.run(ctx, 100000, args.cram_tiles if world == 1 else max(10, args.cram_tiles // 2),
                                          cpu=(world == 1 and not args.no_cpu_baseline))
        except Exception as ex:
            cram = {"error": repr(ex)}
        if world > 1:
            v = [0.0, 0.0, 0.0, 0.0]
            if cram and "records" in cram:
                v = [1.0, cram["slice_decode_ms"] + cram["bam_fill_ms"], cram["e2e_wall_s"], cram.get("encode", {}).get("wall_s", 0.0)]
            tt = torch.tensor(v, dtype=torch.float64, device=dev)
            mn = tt.clone()
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            dist.all_reduce(mn, op=dist.ReduceOp.MIN)
            if cram and "records" in cram and float(mn[0].item()) == 1.0:
                dms, wall, ewall = (float(x) for x in tt[1:].tolist())
                cram.update({"n_gpus": world, "records_per_s_device": world * cram["records"] / dms * 1e3, "records_per_s_e2e": world * cram["records"] / wall,
                             "aggregation": "every rank decodes its own copy; times = max over ranks"})
                if ewall and "records" in cram.get("encode", {}):
                    cram["encode"].update({"wall_s": ewall, "records_per_s_e2e": world * cram["encode"]["records"] / ewall})
            elif cram is not None and "error" not in cram:
                cram = {"error": "a rank failed this leg"}
    if rank != 0:
        return
    hbm, how = peaks()
    achieved = (U + Cb) / ms_step / 1e6
    out = {
        "metric": "BGZF inflate + CRAM rANS decode GB/s at 1/2/4/8 H100 vs reference CPU",
        "value": U * world / ms_step / 1e6, "unit": "GB/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u8", "data": "synthetic",
        "config": {"workload": "BGZF inflate of %.1f GB synthetic 150bp BAM per GPU (30x-shaped, %s 4-bin quals), zlib level %d blocks, one warp per 64 KiB block"
                               % (U / 1e9, args.quals, args.level),
                   "blocks_per_gpu": nb, "uncompressed_bytes_per_gpu": U, "compressed_bytes_per_gpu": Cb,
                   "value_is": "uncompressed bytes / kernel time (inputs resident in HBM)",
                   "l2_policy": "inputs larger than L2 (%.1f GB in + %.1f GB out per step vs 50 MB)" % (Cb / 1e9, U / 1e9),
                   "data_gen_s": round(corpus["gen_s"], 1), "unique_data": "all blocks unique" if corpus["tile"] == 1 else
                                   "%.2f GB unique per GPU repeated %dx at distinct addresses (host cores shared by %d generators)"
                                   % (U / 1e9 / corpus["tile"], corpus["tile"], world)},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": hbm, "unit": "GB/s", "frac": achieved / hbm,
                     "traffic": None, "kernel": "bgzf_inflate_kernel", "algorithmic_bytes_per_launch": U + Cb,
                     "peak_source": how},
        "gpu_launches": int(launches),
        "clocks": clocks,
    }
    if e2e:
        out["e2e"] = e2e
    if bam_extra:
        out.setdefault("extra", {})["bam_unpack"] = bam_extra
    if world == 1 and not args.no_cpu_baseline:
        cb = run_cpu_baseline(corpus, args.cpu_sample_gb)
        if cb:
            out["cpu_baseline"] = cb
    if rans:
        out["rans"] = rans
    if strong:
        out["strong"] = strong
    if numa:
        out["config"]["numa_binding"] = numa
    if world == 1:
        try:
            tl = tok3_leg(args, ctx)
            if tl:
                out.setdefault("extra", {})["tok3_decode"] = tl
        except Exception as ex:
            out.setdefault("extra", {})["tok3_decode"] = {"error": repr(ex)}
    if cram is not None:
        out.setdefault("extra", {})["cram_records"] = cram
    print(json.dumps(out), flush=True)


def tok3_leg(args, ctx):
    """CRAM 3.1 read-name (tok3) blocks, 10 000 names per slice, through the host-buffer API
    (hgpu_tok3_decode_batch_host: framing walk on the host, rANS token streams + name rebuild on the
    device).  Inputs are fixtures written once by the reference encoder (tests/golden/make_tok3_slices.py)."""
    import gzip
    import htslib_b200 as H
    if args.tok3_blocks <= 0:
        return None
    d = os.path.join(ROOT, "tests", "golden", "tok3_slices")
    uniq = [open(os.path.join(d, "slice%d.tok3" % k), "rb").read() for k in range(8)]
    want = [gzip.open(os.path.join(d, "slice%d.names.gz" % k), "rb").read() for k in range(8)]
    Lh = H.lib()
    n = args.tok3_blocks
    comps = [uniq[k % 8] for k in range(n)]
    in_len = np.array([len(c) for c in comps], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.uint64))[:-1]]).astype(np.uint64)
    blob = np.frombuffer(b"".join(comps) + b"\0" * 8, dtype=np.uint8)
    caps = np.array([Lh.hgpu_tok3_out_bound(c, len(c)) for c in comps], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum(caps.astype(np.uint64))[:-1]]).astype(np.uint64)
    out = np.zeros(int(caps.astype(np.uint64).sum()) + 8, dtype=np.uint8)
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    Lh.hgpu_tok3_last_ms.argtypes = [C.c_void_p]
    wall, dev_ms = [], []
    for it in range(1 + 3):
        t0 = time.perf_counter()
        rc = Lh.hgpu_tok3_decode_batch_host(ctx.h, p(blob), p(in_off), p(in_len), n, p(out), p(out_off), p(caps), p(got), p(st))
        t1 = time.perf_counter()
        assert rc == 0, H.last_error()
        ms2 = (C.c_float * 2)()
        Lh.hgpu_tok3_last_ms(ms2)
        if it >= 1:
            wall.append(t1 - t0); dev_ms.append((ms2[0], ms2[1]))
    assert int(np.abs(st).sum()) == 0, "tok3 decode reported errors"
    for k in range(8):
        assert out[int(out_off[k]):int(out_off[k]) + int(got[k])].tobytes() == want[k], "tok3 output differs from the names the fixture was made from"
    U = int(got.astype(np.int64).sum()); Cb = int(in_len.astype(np.int64).sum())
    ent = float(np.mean([a for a, b in dev_ms])); nam = float(np.mean([b for a, b in dev_ms]))
    res = {"workload": "%d tok3 blocks x 10 000 Illumina names (8 unique reference-encoded fixtures tiled), host buffers" % n,
           "blocks": n, "names": n * 10000, "uncompressed_GB": U / 1e9, "compressed_GB": Cb / 1e9,
           "entropy_ms": ent, "rebuild_ms": nam, "device_GBps": U / (ent + nam) / 1e6,
           "names_per_s_device": n * 10000 / ((ent + nam) / 1e3),
           "e2e_ms": float(np.mean(wall)) * 1e3, "e2e_GBps": U / float(np.mean(wall)) / 1e9,
           "unit": "GB/s (uncompressed names)"}
    r = ref_lib()
    if r is not None:                                             # the reference's own decoder, one core, the 8 unique blocks
        r.tok3_decode_names.restype = C.c_void_p
        libc = C.CDLL(None)
        t0 = time.perf_counter(); tot = 0
        for rep in range(3):
            for c in uniq:
                m = C.c_uint(0)
                q = r.tok3_decode_names(c, C.c_uint(len(c)), C.byref(m))
                tot += m.value
                libc.free(C.c_void_p(q))
        res["cpu_reference_1core_GBps"] = tot / (time.perf_counter() - t0) / 1e9
    return res


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    r = ref_lib()
    if r is None:
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/libhts_ref.so was not built (needs /root/reference once)"}))
        return
    corpus = make_corpus(args, 0)
    cores = len(os.sched_getaffinity(0))
    img, ubytes, cbytes, nb = cpu_sample(corpus, args.cpu_sample_gb * 1e9)
    for _ in range(args.warmup):
        ref_decompress(r, img, cores)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        total, _s = ref_decompress(r, img, cores)
        assert total == ubytes
    sec = (time.perf_counter() - t0) / args.steps
    v = ubytes / sec / 1e9
    sample = "first %d BGZF blocks (%.2f GB uncompressed) of the same synthetic BAM per step; unmodified htslib bgzf_read over bgzf_mt(%d), zlib arm (no libdeflate here)" % (nb, ubytes / 1e9, cores)
    print(json.dumps({
        "impl": "reference",
        "metric": "BGZF inflate + CRAM rANS decode GB/s at 1/2/4/8 H100 vs reference CPU",
        "value": v, "unit": "GB/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u8", "data": "synthetic",
        "config": {"workload": "BGZF inflate of synthetic 150bp BAM (same generator as the GPU arm), zlib level %d blocks" % args.level,
                   "sample": sample,
                   "note": "a steady-state rate: each step decodes the first %.1f GB of the same file the GPU arm decodes whole; "
                           "zlib arm of bgzf.c (libdeflate, which htslib recommends and which is roughly 2x faster, is not in this image)" % args.cpu_sample_gb},
        "cpu_baseline": {"value": v, "unit": "GB/s", "cores": cores, "kind": "reference", "sample": sample},
        "e2e": {"value": v, "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            import torch.distributed as dist
            if dist.is_initialized():
                dist.barrier()
                dist.destroy_process_group()
