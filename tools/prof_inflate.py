import sys, ctypes as C, numpy as np, torch, time
sys.path.insert(0,'.'); sys.path.insert(0,'tests')
import htslib_b200 as H
from tools import synth
quals = sys.argv[1] if len(sys.argv)>1 else "novaseq"
corpus = synth.bam_bgzf_corpus(0.5e9, quals=quals)
comp, clen, ulen = corpus["comp"], corpus["clen"], corpus["ulen"]
nb=len(clen); dev=torch.device("cuda:0")
in_off = np.concatenate([[0], np.cumsum(clen.astype(np.int64))[:-1]]).astype(np.uint64)
out_off = np.concatenate([[0], np.cumsum(ulen.astype(np.int64))[:-1]]).astype(np.uint64)
t = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32)).to(dev)
d_in = torch.zeros(comp.size+64, dtype=torch.uint8, device=dev); d_in[:comp.size].copy_(torch.from_numpy(comp.copy()))
d_out = torch.empty(int(ulen.sum())+64, dtype=torch.uint8, device=dev)
a,b,c,d = t(in_off), t(clen), t(out_off), t(ulen)
d_len = torch.zeros(nb, dtype=torch.int32, device=dev); d_st = torch.zeros(nb, dtype=torch.int32, device=dev)
ctx = H.Context(0)
s = torch.cuda.Stream(); torch.cuda.synchronize()
L = H.lib()
buf = (C.c_ulonglong*16)()
with torch.cuda.stream(s):
    for it in range(3):
        L.hgpu_debug_profile(buf)
        e0=torch.cuda.Event(enable_timing=True); e1=torch.cuda.Event(enable_timing=True)
        e0.record(); ctx.bgzf_inflate_dev(d_in,a,b,d_out,c,d,d_len,d_st,s.cuda_stream); e1.record(); torch.cuda.synchronize()
        ms=e0.elapsed_time(e1)
        ok = L.hgpu_debug_profile(buf)
        print(quals, "ms", round(ms,3), "GB/s", round(float(ulen.sum())/ms/1e6,1), "errors", int(d_st.abs().sum()), "prof(cycles/block):", [int(x)//nb for x in buf] if ok==0 else None)
        if ok == 0:
            # counters per block: exec_batch rounds and batches, overlapping matches, the warp's Huffman loop iterations
            # in re-sync round 0 and in the later rounds (warp max per round, summed), iterations of the long-period run path
            per = lambda i: round(int(buf[i]) / nb, 1)
            r0 = per(12)
            print("  rounds", per(8), "batches", per(9), "overlapping", per(11), "resync: round 0", r0, "later rounds", per(13),
                  "(x%.2f of one pass)" % ((r0 + per(13)) / r0 if r0 else 0.0), "long-period run iterations", per(14))
