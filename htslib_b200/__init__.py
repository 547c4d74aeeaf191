"""htslib_b200 — Python face of libhtsgpu.so (hand-written sm_90a CUDA behind a C ABI).

The library is the product; this module only loads it with ctypes and passes raw pointers
(torch is used by callers for device memory and streams, never for compute).  There is no CPU
fallback: if the shared library is missing, importing `htslib_b200.lib()` raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HGPU_LIB") or os.path.join(_HERE, "libhtsgpu.so")   # HGPU_LIB: A/B builds when tuning
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "htsgpu.h")

HGPU_OK = 0
BGZF_ERR_ZLIB, BGZF_ERR_CRC, BGZF_ERR_HEADER, BGZF_ERR_SPACE = -1, -2, -3, -4
RANS_ERR = -1
ERR_ARG = -102
IDX_ERR_READ, IDX_ERR_PUSH = -10, -11

_lib = None
u8p = C.POINTER(C.c_uint8)


class HgpuError(RuntimeError):
    pass


def lib():
    """Load libhtsgpu.so (built in-tree by __graft_entry__.build() / htslib_b200/build.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise HgpuError("libhtsgpu.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`. "
                        "There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32
    L.hgpu_create.restype = vp
    L.hgpu_create.argtypes = [C.c_int]
    L.hgpu_destroy.argtypes = [vp]
    L.hgpu_last_error.restype = C.c_char_p
    L.hgpu_version.restype = C.c_char_p
    L.hgpu_launch_count.restype = u64
    L.hgpu_bgzf_inflate_batch_dev.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp]
    L.hgpu_bgzf_scan.restype = C.c_long
    L.hgpu_bgzf_scan.argtypes = [vp, u64, vp, vp, vp, C.c_long]
    L.hgpu_bgzf_inflate_file_host.argtypes = [vp, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(C.c_long)]
    L.hgpu_bgzf_inflate_blocks_host.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.hgpu_bgzf_compress_batch_dev.argtypes = [vp, vp, vp, vp, u32, C.c_int, vp, vp, vp, vp, vp]
    L.hgpu_shard_range.argtypes = [u64, vp, C.c_int, C.c_int, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.hgpu_crc32.restype = u32
    L.hgpu_crc32.argtypes = [vp, u32, vp, C.c_size_t]
    L.hgpu_rans_nx16_decode_batch_dev.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp]
    L.hgpu_rans_nx16_decode_batch_host.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.hgpu_rans4x8_decode_batch_dev.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp]
    L.hgpu_arith_decode_batch_dev.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp]
    L.hgpu_rans_nx16_wave_size.restype = u32
    L.hgpu_rans_nx16_wave_size.argtypes = [vp]
    L.hgpu_rans_nx16_compress_bound.restype = u32
    L.hgpu_rans_nx16_compress_bound.argtypes = [u32, C.c_int]
    L.hgpu_rans_nx16_encode_batch_dev.argtypes = [vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp]
    L.hgpu_bam_index_records_dev.argtypes = [vp, vp, u64, vp, u64, vp, u64, vp, vp]
    L.hgpu_bam_layout_dev.argtypes = [vp, vp, u64, vp, u64, vp, vp, vp]
    L.hgpu_bam_unpack_dev.argtypes = [vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, vp, vp, vp]
    L.hgpu_bam_pack_dev.argtypes = [vp, vp, vp, vp, u64, vp, vp, vp, vp]
    L.bgzf_compress.argtypes = [vp, C.POINTER(C.c_size_t), vp, C.c_size_t, C.c_int]
    L.rans_uncompress_to_4x16.restype = vp
    L.rans_uncompress_to_4x16.argtypes = [vp, C.c_uint, vp, C.POINTER(C.c_uint)]
    L.rans_uncompress_4x16.restype = vp
    L.rans_uncompress_4x16.argtypes = [vp, C.c_uint, C.POINTER(C.c_uint)]
    L.hts_crc32.restype = u32
    L.hts_crc32.argtypes = [u32, vp, C.c_size_t]
    L.hgpu_tok3_out_bound.restype = u32
    L.hgpu_tok3_out_bound.argtypes = [C.c_char_p, u32]
    L.hgpu_tok3_decode_batch_host.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.tok3_decode_names.restype = vp
    L.tok3_decode_names.argtypes = [C.c_char_p, u32, C.POINTER(u32)]
    _lib = L
    return L


def last_error():
    return lib().hgpu_last_error().decode()


def check(rc, what=""):
    if rc != HGPU_OK:
        raise HgpuError("%s failed: rc=%d (%s)" % (what, rc, last_error()))


class Context:
    """hgpu_ctx wrapper: one device, its streams and scratch."""

    def __init__(self, device=-1):
        self.h = lib().hgpu_create(device)
        if not self.h:
            raise HgpuError("hgpu_create failed: %s" % last_error())

    def close(self):
        if self.h:
            lib().hgpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- device-pointer entry points; tensors are torch CUDA tensors ----
    def bgzf_inflate_dev(self, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, stream=0):
        n = d_in_len.numel()
        check(lib().hgpu_bgzf_inflate_batch_dev(self.h, d_in.data_ptr(), d_in_off.data_ptr(), d_in_len.data_ptr(), n,
                                                d_out.data_ptr(), d_out_off.data_ptr(), d_out_cap.data_ptr(),
                                                d_out_len.data_ptr(), d_status.data_ptr(), stream), "bgzf_inflate_batch_dev")

    def rans_nx16_decode_dev(self, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_len, d_got, d_status, max_out_len, stream=0):
        n = d_in_len.numel()
        check(lib().hgpu_rans_nx16_decode_batch_dev(self.h, d_in.data_ptr(), d_in_off.data_ptr(), d_in_len.data_ptr(), n,
                                                    d_out.data_ptr(), d_out_off.data_ptr(), d_out_len.data_ptr(),
                                                    d_got.data_ptr(), d_status.data_ptr(), int(max_out_len), stream),
              "rans_nx16_decode_batch_dev")

    def tok3_decode(self, comps):
        """Decode a list of tok3 name blocks (host buffers); returns list of (status, bytes)."""
        import numpy as np
        L = lib()
        n = len(comps)
        in_len = np.array([len(c) for c in comps], dtype=np.uint32)
        in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.uint64))[:-1]]).astype(np.uint64)
        blob = np.frombuffer(b"".join(comps) + b"\0" * 8, dtype=np.uint8)
        caps = np.array([max(1024, L.hgpu_tok3_out_bound(bytes(c), len(c))) for c in comps], dtype=np.uint32)
        out_off = np.concatenate([[0], np.cumsum(caps.astype(np.uint64))[:-1]]).astype(np.uint64)
        out = np.zeros(int(caps.astype(np.uint64).sum()) + 8, dtype=np.uint8)
        got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        check(L.hgpu_tok3_decode_batch_host(self.h, p(blob), p(in_off), p(in_len), n, p(out), p(out_off), p(caps), p(got), p(st)),
              "tok3_decode_batch_host")
        return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]

    def arith_decode(self, comps, caps, stream=0):
        """Decode a list of arith_dynamic streams on the device; returns list of (status, bytes)."""
        return self._decode_list(lib().hgpu_arith_decode_batch_dev, comps, caps, stream, True)

    def _decode_list(self, fn, comps, caps, stream, with_max):
        import numpy as np
        import torch
        n = len(comps)
        dev = torch.device("cuda", torch.cuda.current_device())
        in_len = np.array([len(c) for c in comps], dtype=np.uint32)
        in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64) + 3)[:-1]]).astype(np.int64)
        blob = np.zeros(int(in_off[-1]) + int(in_len[-1]) + 8, dtype=np.uint8)
        for o, c in zip(in_off, comps):
            blob[int(o):int(o) + len(c)] = np.frombuffer(c, dtype=np.uint8)
        out_len = np.array(caps, dtype=np.uint32)
        out_off = np.concatenate([[0], np.cumsum(out_len.astype(np.int64) + 1)[:-1]]).astype(np.int64)
        t = lambda a: torch.from_numpy(a).to(dev)
        d_in = t(blob); d_out = torch.zeros(int(out_off[-1]) + int(out_len[-1]) + 8, dtype=torch.uint8, device=dev)
        d_io, d_il, d_oo, d_ol = t(in_off), t(in_len.view(np.int32)), t(out_off), t(out_len.view(np.int32))
        d_got = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
        args = [self.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), n, d_out.data_ptr(), d_oo.data_ptr(),
                d_ol.data_ptr(), d_got.data_ptr(), d_st.data_ptr()]
        if with_max:
            args.append(int(out_len.max()) if n else 0)
        args.append(stream)
        check(fn(*args), "decode batch")
        torch.cuda.synchronize()
        out = d_out.cpu().numpy(); got = d_got.cpu().numpy(); st = d_st.cpu().numpy()
        return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]

    def rans4x8_decode(self, comps, caps, stream=0):
        """Decode a list of rANS 4x8 streams on the device; returns list of (status, bytes)."""
        import numpy as np
        import torch
        n = len(comps)
        dev = torch.device("cuda", torch.cuda.current_device())
        in_len = np.array([len(c) for c in comps], dtype=np.uint32)
        in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64) + 3)[:-1]]).astype(np.int64)
        blob = np.zeros(int(in_off[-1]) + int(in_len[-1]) + 8, dtype=np.uint8)
        for o, c in zip(in_off, comps):
            blob[int(o):int(o) + len(c)] = np.frombuffer(c, dtype=np.uint8)
        out_len = np.array(caps, dtype=np.uint32)
        out_off = np.concatenate([[0], np.cumsum(out_len.astype(np.int64) + 1)[:-1]]).astype(np.int64)
        t = lambda a: torch.from_numpy(a).to(dev)
        d_in = t(blob); d_out = torch.zeros(int(out_off[-1]) + int(out_len[-1]) + 8, dtype=torch.uint8, device=dev)
        d_io, d_il, d_oo, d_ol = t(in_off), t(in_len.view(np.int32)), t(out_off), t(out_len.view(np.int32))
        d_got = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
        check(lib().hgpu_rans4x8_decode_batch_dev(self.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), n, d_out.data_ptr(),
                                                  d_oo.data_ptr(), d_ol.data_ptr(), d_got.data_ptr(), d_st.data_ptr(), stream),
              "rans4x8_decode_batch_dev")
        torch.cuda.synchronize()
        out = d_out.cpu().numpy(); got = d_got.cpu().numpy(); st = d_st.cpu().numpy()
        return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]

    def bgzf_compress(self, payloads, level=6, stream=0):
        """Compress a list of payloads (each <= 65280 bytes) into BGZF blocks on the device."""
        import numpy as np
        import torch
        n = len(payloads)
        dev = torch.device("cuda", torch.cuda.current_device())
        in_len = np.array([len(p) for p in payloads], dtype=np.uint32)
        in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64))[:-1]]).astype(np.int64)
        blob = np.frombuffer(b"".join(payloads) + b"\0" * 8, dtype=np.uint8).copy()
        d_in = torch.from_numpy(blob).to(dev)
        d_out = torch.zeros(n * 65536 + 64, dtype=torch.uint8, device=dev)
        out_off = np.arange(n, dtype=np.int64) * 65536
        t = lambda a: torch.from_numpy(a).to(dev)
        d_io, d_il, d_oo = t(in_off), t(in_len.view(np.int32)), t(out_off)
        d_ol = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
        check(lib().hgpu_bgzf_compress_batch_dev(self.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), n, level,
                                                 d_out.data_ptr(), d_oo.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), stream),
              "bgzf_compress_batch_dev")
        torch.cuda.synchronize()
        out = d_out.cpu().numpy(); ol = d_ol.cpu().numpy(); st = d_st.cpu().numpy()
        return [out[i * 65536:i * 65536 + int(ol[i])].tobytes() if st[i] == 0 else None for i in range(n)]

    def rans_nx16_encode(self, raws, orders, stream=0):
        """Encode a list of byte strings on the device (hgpu_rans_nx16_encode_batch_dev).  Returns
        list of compressed byte strings (None where the kernel reported failure)."""
        import numpy as np
        import torch
        L = lib()
        n = len(raws)
        dev = torch.device("cuda", torch.cuda.current_device())
        in_len = np.array([len(r) for r in raws], dtype=np.uint32)
        in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64))[:-1]]).astype(np.int64)
        cap = np.array([L.hgpu_rans_nx16_compress_bound(int(l), int(o)) for l, o in zip(in_len, orders)], dtype=np.uint32)
        out_off = np.concatenate([[0], np.cumsum((cap.astype(np.int64) + 15) // 16 * 16)[:-1]]).astype(np.int64)
        blob = np.frombuffer(b"".join(raws) + b"\0" * 8, dtype=np.uint8).copy()
        d_in = torch.from_numpy(blob).to(dev)
        d_out = torch.zeros(int(out_off[-1]) + int(cap[-1]) + 64, dtype=torch.uint8, device=dev)
        t = lambda a: torch.from_numpy(a).to(dev)
        d_io, d_il, d_or = t(in_off), t(in_len.view(np.int32)), t(np.array(orders, dtype=np.int32))
        d_oo, d_oc = t(out_off), t(cap.view(np.int32))
        d_ol = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
        check(L.hgpu_rans_nx16_encode_batch_dev(self.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), d_or.data_ptr(), n,
                                                d_out.data_ptr(), d_oo.data_ptr(), d_oc.data_ptr(), d_ol.data_ptr(),
                                                d_st.data_ptr(), stream), "rans_nx16_encode_batch_dev")
        torch.cuda.synchronize()
        out = d_out.cpu().numpy(); ol = d_ol.cpu().numpy(); st = d_st.cpu().numpy()
        return [out[int(o):int(o) + int(l)].tobytes() if s == 0 else None for o, l, s in zip(out_off, ol, st)]

    def bam_unpack_dev(self, d_stream, length, d_hint=None, want_text=True, stream=0):
        """index -> layout -> unpack of an inflated BAM record stream resident on the device.
        Returns dict of torch tensors: rec_off, core (n x 48 bytes), data, data_off, seq, qual, seq_off, status."""
        import torch
        dev = d_stream.device
        L = lib()
        d_n = torch.zeros(1, dtype=torch.int64, device=dev)
        nh = d_hint.numel() if d_hint is not None else 0
        hp = d_hint.data_ptr() if d_hint is not None else None
        check(L.hgpu_bam_index_records_dev(self.h, d_stream.data_ptr(), length, hp, nh, None, 0, d_n.data_ptr(), stream), "bam_index(count)")
        torch.cuda.synchronize()
        n = int(d_n.item())
        if n < 0:
            raise HgpuError("malformed BAM record chain")
        rec_off = torch.empty(max(1, n), dtype=torch.int64, device=dev)
        check(L.hgpu_bam_index_records_dev(self.h, d_stream.data_ptr(), length, hp, nh, rec_off.data_ptr(), n, d_n.data_ptr(), stream), "bam_index")
        data_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        seq_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        check(L.hgpu_bam_layout_dev(self.h, d_stream.data_ptr(), length, rec_off.data_ptr(), n, data_off.data_ptr(), seq_off.data_ptr(), stream), "bam_layout")
        torch.cuda.synchronize()
        nd, ns = int(data_off[n].item()), int(seq_off[n].item())
        core = torch.empty((max(1, n), 48), dtype=torch.uint8, device=dev)
        data = torch.empty(max(1, nd), dtype=torch.uint8, device=dev)
        seq = torch.empty(max(1, ns), dtype=torch.uint8, device=dev) if want_text else None
        qual = torch.empty(max(1, ns), dtype=torch.uint8, device=dev) if want_text else None
        status = torch.empty(max(1, n), dtype=torch.int32, device=dev)
        check(L.hgpu_bam_unpack_dev(self.h, d_stream.data_ptr(), length, rec_off.data_ptr(), n, core.data_ptr(), data.data_ptr(),
                                    data_off.data_ptr(), seq.data_ptr() if want_text else None, qual.data_ptr() if want_text else None,
                                    seq_off.data_ptr(), status.data_ptr(), stream), "bam_unpack")
        return dict(n=n, rec_off=rec_off, core=core, data=data, data_off=data_off, seq=seq, qual=qual, seq_off=seq_off, status=status)

    def sam_format_dev(self, core, data, data_off, n, target_names, stream=0):
        """SAM text lines (sam_format1 + newline) of n unpacked records on the device (hgpu_sam_format_dev).
        target_names: list of bytes (the header's @SQ names).  Returns (text uint8 tensor, out_off int64[n+1], status)."""
        import numpy as np
        import torch
        dev = core.device
        L = lib()
        L.hgpu_sam_format_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        blob = b"".join(target_names) + b"\0"
        noff = np.concatenate([[0], np.cumsum([len(x) for x in target_names])]).astype(np.int64)
        d_names = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).to(dev)
        d_noff = torch.from_numpy(noff).to(dev)
        out_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        status = torch.zeros(max(1, n), dtype=torch.int32, device=dev)
        args = (self.h, core.data_ptr(), data.data_ptr(), data_off.data_ptr(), n, d_names.data_ptr(), d_noff.data_ptr(), len(target_names))
        check(L.hgpu_sam_format_dev(*args, None, out_off.data_ptr(), status.data_ptr(), stream), "sam_format(layout)")
        torch.cuda.synchronize()
        total = int(out_off[n].item())
        out = torch.empty(max(1, total), dtype=torch.uint8, device=dev)
        check(L.hgpu_sam_format_dev(*args, out.data_ptr(), out_off.data_ptr(), None, stream), "sam_format")
        return out[:total], out_off, status

    def bam_pack_dev(self, core, data, data_off, n, stream=0):
        """bam_write1 data movement on the device: returns (out uint8 tensor, out_off int64[n+1], status)."""
        import torch
        dev = core.device
        out_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        status = torch.zeros(max(1, n), dtype=torch.int32, device=dev)
        L = lib()
        check(L.hgpu_bam_pack_dev(self.h, core.data_ptr(), data.data_ptr(), data_off.data_ptr(), n, None, out_off.data_ptr(), None, stream), "bam_pack(layout)")
        torch.cuda.synchronize()
        total = int(out_off[n].item())
        out = torch.empty(max(1, total), dtype=torch.uint8, device=dev)
        check(L.hgpu_bam_pack_dev(self.h, core.data_ptr(), data.data_ptr(), data_off.data_ptr(), n, out.data_ptr(), out_off.data_ptr(), status.data_ptr(), stream), "bam_pack")
        return out[:total], out_off, status

    # ---- host-pointer entry points; buffers are numpy uint8 arrays (or pinned torch tensors' .numpy()) ----
    def bgzf_inflate_file_host(self, file_np, out_np):
        out_len = C.c_uint64(0)
        bad = C.c_long(-1)
        rc = lib().hgpu_bgzf_inflate_file_host(self.h, file_np.ctypes.data, file_np.size, out_np.ctypes.data, out_np.size,
                                               C.byref(out_len), C.byref(bad))
        return rc, out_len.value, bad.value

    def bam_index(self, file_np, min_shift=0, window_bytes=0):
        """The BAI (min_shift <= 0) or CSI (min_shift > 0) file of a whole BAM image, as sam_index_build3 writes it
        (hgpu_bam_index_build_host).  Raises HgpuError with .code and .bad (the refused record, or the bad block)."""
        L = lib()
        L.hgpu_bam_index_build_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint64,
                                                C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
        L.hgpu_bam_index_build_host.restype = C.c_int
        out, n, bad = C.c_void_p(), C.c_uint64(0), C.c_int64(-1)
        rc = L.hgpu_bam_index_build_host(self.h, file_np.ctypes.data, file_np.size, min_shift, window_bytes,
                                         C.byref(out), C.byref(n), C.byref(bad))
        if rc != HGPU_OK:
            e = HgpuError("bam_index failed: rc=%d bad=%d (%s)" % (rc, bad.value, last_error()))
            e.code, e.bad = rc, bad.value
            raise e
        try:
            return C.string_at(out, n.value)
        finally:
            libc = C.CDLL(None)
            libc.free.argtypes = [C.c_void_p]
            libc.free(out)

    def bam_index_last_ms(self):
        """(device ms of the windows, host finishing ms) of the last bam_index call."""
        ms = (C.c_float * 2)()
        lib().hgpu_bam_index_last_ms(ms)
        return ms[0], ms[1]

    def cram_index(self, file_np):
        """The .crai file of a whole CRAM 3.x image, as sam_index_build3 writes it (hgpu_cram_index_build_host): one gzip
        member.  Raises HgpuError with .code and .bad (the slice, in file order, where the reference stops)."""
        L = lib()
        L.hgpu_cram_index_build_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                                 C.POINTER(C.c_int64)]
        L.hgpu_cram_index_build_host.restype = C.c_int
        out, n, bad = C.c_void_p(), C.c_uint64(0), C.c_int64(-1)
        rc = L.hgpu_cram_index_build_host(self.h, file_np.ctypes.data, file_np.size, C.byref(out), C.byref(n), C.byref(bad))
        if rc != HGPU_OK:
            e = HgpuError("cram_index failed: rc=%d bad=%d (%s)" % (rc, bad.value, last_error()))
            e.code, e.bad = rc, bad.value
            raise e
        try:
            return C.string_at(out, n.value)
        finally:
            libc = C.CDLL(None)
            libc.free.argtypes = [C.c_void_p]
            libc.free(out)

    def cram_index_last_ms(self):
        """(device ms of the slice decode and runs kernels, ms of the rest of the call) of the last cram_index call."""
        ms = (C.c_float * 2)()
        lib().hgpu_cram_index_last_ms(ms)
        return ms[0], ms[1]

    def rans_nx16_decode_host(self, in_np, in_off, in_len, out_np, out_off, out_len):
        import numpy as np
        n = len(in_len)
        got = np.zeros(n, dtype=np.uint32)
        st = np.zeros(n, dtype=np.int32)
        check(lib().hgpu_rans_nx16_decode_batch_host(self.h, in_np.ctypes.data, in_off.ctypes.data, in_len.ctypes.data, n,
                                                     out_np.ctypes.data, out_off.ctypes.data, out_len.ctypes.data,
                                                     got.ctypes.data, st.ctypes.data), "rans_nx16_decode_batch_host")
        return got, st

    def crc32(self, data, crc=0):
        import numpy as np
        a = np.frombuffer(data, dtype=np.uint8)
        return lib().hgpu_crc32(self.h, crc, a.ctypes.data if a.size else None, a.size)


def shard_range(unit_out_len, world, rank):
    """(first, count, out_base) of this rank's contiguous unit range (hgpu_shard_range)."""
    import numpy as np
    a = np.ascontiguousarray(unit_out_len, dtype=np.uint32)
    f, c, b = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    check(lib().hgpu_shard_range(a.size, a.ctypes.data, world, rank, C.byref(f), C.byref(c), C.byref(b)), "shard_range")
    return f.value, c.value, b.value


def cram_scan_blocks(file_np):
    """List the blocks of a CRAM 3.x file image: structured numpy array (hgpu_cram_block)."""
    import numpy as np
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"),
                   ("method", "u1"), ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])
    assert dt.itemsize == 32
    L = lib()
    L.hgpu_cram_scan_blocks.restype = C.c_long
    L.hgpu_cram_scan_blocks.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    maj, mnr = C.c_int(0), C.c_int(0)
    n = L.hgpu_cram_scan_blocks(file_np.ctypes.data, file_np.size, None, 0, C.byref(maj), C.byref(mnr))
    if n < 0:
        raise HgpuError("CRAM scan failed: %s" % last_error())
    arr = np.zeros(n, dtype=dt)
    L.hgpu_cram_scan_blocks(file_np.ctypes.data, file_np.size, arr.ctypes.data, n, C.byref(maj), C.byref(mnr))
    return arr, (maj.value, mnr.value)


class CramRefs(C.Structure):
    _fields_ = [("bases", C.c_void_p), ("off", C.c_void_p), ("n_ref", C.c_int32)]


class CramRecords(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("data_bytes", C.c_uint64), ("n_slices", C.c_uint32), ("pad", C.c_uint32),
                ("core", C.c_void_p), ("data", C.c_void_p), ("data_off", C.c_void_p),
                ("rec_status", C.c_void_p), ("slice_status", C.c_void_p), ("slice_rec0", C.c_void_p)]


BAM1_CORE_DT = [("pos", "<i8"), ("tid", "<i4"), ("bin", "<u2"), ("qual", "u1"), ("l_extranul", "u1"), ("flag", "<u2"), ("l_qname", "<u2"),
                ("n_cigar", "<u4"), ("l_qseq", "<i4"), ("mtid", "<i4"), ("mpos", "<i8"), ("isize", "<i8")]


def cram_sq_names(blocks, udata, udata_off):
    """@SQ SN names of a CRAM file, from its (uncompressed) file header block."""
    import struct
    i = [k for k in range(len(blocks)) if int(blocks[k]["content_type"]) == 0][0]
    o = int(udata_off[i])
    n = struct.unpack("<i", udata[o:o + 4].tobytes())[0]
    text = udata[o + 4:o + 4 + n].tobytes()
    return [[f[3:] for f in line.split(b"\t") if f.startswith(b"SN:")][0] for line in text.split(b"\n") if line.startswith(b"@SQ\t")]


def load_fasta_upper(path, names=None):
    """Reference sequences of a FASTA file, upper case (what cram_get_ref hands the decoder, cram/cram_io.c:3270-3310), in file
    order or in the order of `names` (the header's @SQ lines; a name the file lacks gets an empty sequence):
    returns (bases uint8 array, offsets uint64 array of n + 1)."""
    import numpy as np
    seqs, cur, order = {}, None, []
    for line in open(path, "rb"):
        if line.startswith(b">"):
            cur = []
            nm = line[1:].split()[0]
            seqs[nm] = cur
            order.append(nm)
        elif cur is not None:
            cur.append(line.strip())
    flat = [np.frombuffer(b"".join(seqs.get(nm, [])), dtype=np.uint8) & 0xdf for nm in (names if names is not None else order)]
    off = np.zeros(len(flat) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(f) for f in flat])
    return (np.concatenate(flat) if flat else np.zeros(0, dtype=np.uint8)), off


def _records_out(out, free):
    import numpy as np
    n, ns = out.n_records, out.n_slices
    def arr(ptr, count, dt):
        if not count:
            return np.zeros(0, dtype=dt)
        return np.frombuffer((C.c_uint8 * (count * np.dtype(dt).itemsize)).from_address(ptr), dtype=dt).copy()
    core = arr(out.core, n, np.dtype(BAM1_CORE_DT))
    doff = arr(out.data_off, n + 1, np.uint64)
    blob = arr(out.data, out.data_bytes, np.uint8).tobytes()
    res = {"core": core, "data": [blob[int(doff[i]):int(doff[i + 1])] for i in range(n)], "rec_status": arr(out.rec_status, n, np.int32),
           "slice_status": arr(out.slice_status, ns, np.int32), "slice_rec0": arr(out.slice_rec0, ns + 1, np.uint64)}
    free.argtypes = [C.c_void_p]
    free(C.byref(out))
    return res


def cram_decode_file(ctx, file_np, fasta=None, prefix=b"", decode_md=0):
    """hgpu_cram_decode_file_host: scan + uncompress + record decode of a CRAM file image in one call."""
    import numpy as np
    L = lib()
    refs = CramRefs()
    keep = None
    if fasta is not None:
        keep = (np.ascontiguousarray(fasta[0]), np.ascontiguousarray(fasta[1]))
        refs.bases = keep[0].ctypes.data; refs.off = keep[1].ctypes.data; refs.n_ref = len(keep[1]) - 1
    out = CramRecords()
    L.hgpu_cram_decode_file_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
    rc = L.hgpu_cram_decode_file_host(ctx.h, file_np.ctypes.data, file_np.size, C.byref(refs) if fasta is not None else None, prefix, decode_md, C.byref(out))
    if rc != 0:
        raise HgpuError("cram_decode_file: %d %s" % (rc, last_error()))
    return _records_out(out, L.hgpu_cram_records_free)


class CramRecordsDev(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("data_bytes", C.c_uint64), ("d_core", C.c_void_p), ("d_data", C.c_void_p),
                ("d_data_off", C.c_void_p), ("d_rec_status", C.c_void_p)]


def cram_decode_records_dev(ctx, file_np, blocks, udata, udata_off, fasta=None, prefix=b"", decode_md=0):
    """hgpu_cram_decode_records_dev: the records stay in HBM.  Returns (CramRecordsDev with raw device pointers, slice_status)."""
    import numpy as np
    L = lib()
    refs = CramRefs()
    keep = None
    if fasta is not None:
        keep = (np.ascontiguousarray(fasta[0]), np.ascontiguousarray(fasta[1]))
        refs.bases = keep[0].ctypes.data; refs.off = keep[1].ctypes.data; refs.n_ref = len(keep[1]) - 1
    out, dev = CramRecords(), CramRecordsDev()
    L.hgpu_cram_decode_records_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]
    rc = L.hgpu_cram_decode_records_dev(ctx.h, file_np.ctypes.data, file_np.size, blocks.ctypes.data, len(blocks), udata.ctypes.data,
                                        udata_off.ctypes.data, C.byref(refs) if fasta is not None else None, prefix, decode_md,
                                        C.byref(out), C.byref(dev))
    if rc != 0:
        raise HgpuError("cram_decode_records_dev: %d %s" % (rc, last_error()))
    ns = out.n_slices
    sst = np.frombuffer((C.c_uint8 * (ns * 4)).from_address(out.slice_status), dtype=np.int32).copy() if ns else np.zeros(0, dtype=np.int32)
    L.hgpu_cram_records_free.argtypes = [C.c_void_p]
    L.hgpu_cram_records_free(C.byref(out))
    return dev, sst


def cram_decode_records(ctx, file_np, blocks, udata, udata_off, fasta=None, prefix=b"", decode_md=0, _entry=None):
    """Every record of a CRAM 3.x image as bam1_t (hgpu_cram_decode_records_host).  udata / udata_off: the blocks
    uncompressed (cram_uncompress_blocks).  fasta: (bases, offsets) from load_fasta_upper, or None.
    Returns dict: core (structured array), data (list of bytes), rec_status, slice_status, slice_rec0."""
    import numpy as np
    L = lib()
    refs = CramRefs()
    keep = None
    if fasta is not None:
        keep = (np.ascontiguousarray(fasta[0]), np.ascontiguousarray(fasta[1]))
        refs.bases = keep[0].ctypes.data; refs.off = keep[1].ctypes.data; refs.n_ref = len(keep[1]) - 1
    out = CramRecords()
    if _entry is None:
        L.hgpu_cram_decode_records_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
        rc = L.hgpu_cram_decode_records_host(ctx.h, file_np.ctypes.data, file_np.size, blocks.ctypes.data, len(blocks), udata.ctypes.data,
                                             udata_off.ctypes.data, C.byref(refs) if fasta is not None else None, prefix, decode_md, C.byref(out))
        free, err = L.hgpu_cram_records_free, last_error
    else:
        fn, free, err = _entry
        rc = fn(file_np.ctypes.data, file_np.size, blocks.ctypes.data, len(blocks), udata.ctypes.data, udata_off.ctypes.data,
                C.byref(refs) if fasta is not None else None, prefix, decode_md, C.byref(out))
    if rc != 0:
        raise HgpuError("cram_decode_records: %d %s" % (rc, err()))
    return _records_out(out, free)


CRAM_ENC_ATTACH_MATES = 0x1          # HGPU_CRAM_ENC_ATTACH_MATES
CRAM_ENC_TAG_BLOCKS = 0x2            # HGPU_CRAM_ENC_TAG_BLOCKS


def cram_encode_records(ctx, header_text, core, data, data_off, n, fasta=None, records_per_slice=0, minor_version=1, enc_flags=0):
    """hgpu_cram_encode_records_opts_host: n bam1_t records (core: BAM1_CORE_DT array, data: uint8, data_off: uint64 n + 1)
    -> a CRAM 3.x file image (bytes).  fasta: load_fasta_upper's (bases, offsets) in @SQ order, or None."""
    L = lib()
    refs, keep = _cram_refs(fasta)
    L.hgpu_cram_encode_records_opts_host.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                                     C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p]
    out, ln = C.c_void_p(), C.c_uint64(0)
    rc = L.hgpu_cram_encode_records_opts_host(ctx.h, header_text, len(header_text), core.ctypes.data, data.ctypes.data, data_off.ctypes.data, n,
                                              refs, records_per_slice, minor_version, enc_flags, C.byref(out), C.byref(ln))
    if rc != 0:
        raise HgpuError("cram_encode_records: %d %s" % (rc, last_error()))
    img = C.string_at(out.value, ln.value)
    C.CDLL(None).free(C.c_void_p(out.value))
    return img


def cram_encode_last_ms():
    """(pairing kernels, count + scan + write kernels) device ms of the last cram_encode_records call."""
    a, b = C.c_float(0), C.c_float(0)
    lib().hgpu_cram_encode_last_ms(C.byref(a), C.byref(b))
    return a.value, b.value


def cram_encode_tags_last_ms():
    """Device ms of the tag pass of the last cram_encode_records call (0 when it did not run)."""
    a = C.c_float(0)
    lib().hgpu_cram_encode_tags_last_ms(C.byref(a))
    return a.value


# CRAM_OPT_REQUIRED_FIELDS bits (htslib's SAM_*, hts.h:279-291; HGPU_SAM_* in htsgpu.h)
SAM_QNAME, SAM_FLAG, SAM_RNAME, SAM_POS, SAM_MAPQ, SAM_CIGAR, SAM_RNEXT = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40
SAM_PNEXT, SAM_TLEN, SAM_SEQ, SAM_QUAL, SAM_AUX, SAM_RGAUX, SAM_ALL = 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x7fffffff


def _cram_refs(fasta):
    """(CramRefs pointer or None, arrays to keep alive) for load_fasta_upper's (bases, offsets)."""
    import numpy as np
    if fasta is None:
        return None, None
    keep = (np.ascontiguousarray(fasta[0]), np.ascontiguousarray(fasta[1]))
    refs = CramRefs()
    refs.bases = keep[0].ctypes.data; refs.off = keep[1].ctypes.data; refs.n_ref = len(keep[1]) - 1
    return C.byref(refs), (keep, refs)


def cram_required_blocks(blocks, udata, udata_off, required_fields, _entry=None):
    """hgpu_cram_required_blocks: uint8 array, 1 for every block a decode of `required_fields` reads.  Only the header
    blocks (content types 0 / 1 / 2) of udata need to be uncompressed.  _entry: (function, error) of another build."""
    import numpy as np
    used = np.zeros(len(blocks) + 1, dtype=np.uint8)
    barr = np.ascontiguousarray(blocks)
    if _entry is None:
        L = lib()
        fn, err = L.hgpu_cram_required_blocks, last_error
    else:
        fn, err = _entry
    fn.restype = C.c_long
    fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    n = fn(barr.ctypes.data, len(blocks), udata.ctypes.data, udata_off.ctypes.data, required_fields, used.ctypes.data)
    if n < 0:
        raise HgpuError("cram_required_blocks: %s" % err())
    return used[:len(blocks)]


def cram_decode_records_fields(ctx, file_np, blocks, udata, udata_off, fasta=None, prefix=b"", decode_md=0, required_fields=0, _entry=None):
    """cram_decode_records for a field subset (hgpu_cram_decode_records_fields_host): what sam_read1 returns after
    hts_set_opt(CRAM_OPT_REQUIRED_FIELDS, required_fields).  Blocks cram_required_blocks marks unused may hold anything.
    _entry: (function, free, error) of another build of the same entry point (tests/hostsim)."""
    refs, keep = _cram_refs(fasta)
    out = CramRecords()
    if _entry is None:
        L = lib()
        fn, free, err = L.hgpu_cram_decode_records_fields_host, L.hgpu_cram_records_free, last_error
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int,
                       C.c_uint32, C.c_void_p]
        rc = fn(ctx.h, file_np.ctypes.data, file_np.size, blocks.ctypes.data, len(blocks), udata.ctypes.data, udata_off.ctypes.data, refs,
                prefix, decode_md, required_fields, C.byref(out))
    else:
        fn, free, err = _entry
        rc = fn(file_np.ctypes.data, file_np.size, blocks.ctypes.data, len(blocks), udata.ctypes.data, udata_off.ctypes.data, refs,
                prefix, decode_md, required_fields, C.byref(out))
    if rc != 0:
        raise HgpuError("cram_decode_records_fields: %d %s" % (rc, err()))
    return _records_out(out, free)


def cram_decode_file_fields(ctx, file_np, fasta=None, prefix=b"", decode_md=0, required_fields=0):
    """hgpu_cram_decode_file_fields_host: scan, uncompress only the blocks the fields need, decode those fields."""
    L = lib()
    refs, keep = _cram_refs(fasta)
    out = CramRecords()
    L.hgpu_cram_decode_file_fields_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_uint32, C.c_void_p]
    rc = L.hgpu_cram_decode_file_fields_host(ctx.h, file_np.ctypes.data, file_np.size, refs, prefix, decode_md, required_fields, C.byref(out))
    if rc != 0:
        raise HgpuError("cram_decode_file_fields: %d %s" % (rc, last_error()))
    return _records_out(out, L.hgpu_cram_records_free)


def bgzf_scan(file_np):
    """BSIZE-chain walk: returns (off u64[n], len u32[n], isize u32[n]) or raises on a bad block."""
    import numpy as np
    n = lib().hgpu_bgzf_scan(file_np.ctypes.data, file_np.size, None, None, None, 0)
    if n < 0:
        raise HgpuError("bad BGZF block %d" % (-1 - n))
    off = np.zeros(n, dtype=np.uint64); ln = np.zeros(n, dtype=np.uint32); isz = np.zeros(n, dtype=np.uint32)
    lib().hgpu_bgzf_scan(file_np.ctypes.data, file_np.size, off.ctypes.data, ln.ctypes.data, isz.ctypes.data, n)
    return off, ln, isz


def cram_uncompress_blocks(ctx, file_np, blocks=None):
    """Uncompress every block of a CRAM file image on the device (hgpu_cram_uncompress_blocks_host).
    Returns (blocks, [(status, bytes)])."""
    import numpy as np
    if blocks is None:
        blocks, _ = cram_scan_blocks(file_np)
    n = len(blocks)
    sizes = blocks["uncomp_size"].astype(np.uint64)
    out_off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)[:-1]]).astype(np.uint64) if n else np.zeros(0, np.uint64)
    out = np.zeros(int(out_off[-1] + sizes[-1]) + 16 if n else 16, dtype=np.uint8)
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    L = lib()
    L.hgpu_cram_uncompress_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
    barr = np.ascontiguousarray(blocks)
    check(L.hgpu_cram_uncompress_blocks_host(ctx.h, file_np.ctypes.data, file_np.size, barr.ctypes.data, n, out.ctypes.data,
                                             out_off.ctypes.data, got.ctypes.data, st.ctypes.data), "cram_uncompress_blocks_host")
    return blocks, [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]


def fqz_decode(ctx, comps, caps):
    """Decode a list of fqzcomp quality streams (hgpu_fqz_decode_batch_host); returns [(status, bytes)]."""
    import numpy as np
    L = lib()
    L.hgpu_fqz_decode_batch_host.argtypes = [C.c_void_p] * 4 + [C.c_uint32] + [C.c_void_p] * 5
    n = len(comps)
    in_len = np.array([len(c) for c in comps], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.uint64))[:-1]]).astype(np.uint64)
    blob = np.frombuffer(b"".join(comps) + b"\0" * 8, dtype=np.uint8)
    cap = np.array(caps, dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum((cap.astype(np.uint64) + 15) // 16 * 16)[:-1]]).astype(np.uint64)
    out = np.zeros(int(out_off[-1] + cap[-1]) + 16, dtype=np.uint8)
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    check(L.hgpu_fqz_decode_batch_host(ctx.h, p(blob), p(in_off), p(in_len), n, p(out), p(out_off), p(cap), p(got), p(st)),
          "fqz_decode_batch_host")
    return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]


def arith_encode(ctx, raws, orders, stream=0):
    """Encode byte strings with the adaptive arithmetic coder on the device (hgpu_arith_encode_batch_dev).
    Returns the compressed byte strings (None where the kernel reported failure)."""
    import numpy as np
    import torch
    L = lib()
    L.hgpu_arith_compress_bound.restype = C.c_uint32
    L.hgpu_arith_compress_bound.argtypes = [C.c_uint32, C.c_int]
    L.hgpu_arith_encode_batch_dev.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p]
    n = len(raws)
    dev = torch.device("cuda", torch.cuda.current_device())
    in_len = np.array([len(r) for r in raws], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64))[:-1]]).astype(np.int64)
    cap = np.array([L.hgpu_arith_compress_bound(int(l), int(o)) for l, o in zip(in_len, orders)], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum((cap.astype(np.int64) + 15) // 16 * 16)[:-1]]).astype(np.int64)
    blob = np.frombuffer(b"".join(raws) + b"\0" * 8, dtype=np.uint8).copy()
    d_in = torch.from_numpy(blob).to(dev)
    d_out = torch.zeros(int(out_off[-1]) + int(cap[-1]) + 64, dtype=torch.uint8, device=dev)
    t = lambda a: torch.from_numpy(a).to(dev)
    d_io, d_il, d_or = t(in_off), t(in_len.view(np.int32)), t(np.array(orders, dtype=np.int32))
    d_oo, d_oc = t(out_off), t(cap.view(np.int32))
    d_ol = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
    check(L.hgpu_arith_encode_batch_dev(ctx.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), d_or.data_ptr(), n,
                                        d_out.data_ptr(), d_oo.data_ptr(), d_oc.data_ptr(), d_ol.data_ptr(),
                                        d_st.data_ptr(), int(in_len.max()) if n else 0, stream), "arith_encode_batch_dev")
    torch.cuda.synchronize()
    out = d_out.cpu().numpy(); ol = d_ol.cpu().numpy(); st = d_st.cpu().numpy()
    return [out[int(o):int(o) + int(l)].tobytes() if s == 0 else None for o, l, s in zip(out_off, ol, st)]


def _encode_list(ctx, fn, bound, raws, orders, stream, extra=()):
    import numpy as np
    import torch
    n = len(raws)
    dev = torch.device("cuda", torch.cuda.current_device())
    in_len = np.array([len(r) for r in raws], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.int64))[:-1]]).astype(np.int64)
    cap = np.array([bound(int(l), int(o)) for l, o in zip(in_len, orders)], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum((cap.astype(np.int64) + 15) // 16 * 16)[:-1]]).astype(np.int64)
    blob = np.frombuffer(b"".join(raws) + b"\0" * 8, dtype=np.uint8).copy()
    d_in = torch.from_numpy(blob).to(dev)
    d_out = torch.zeros(int(out_off[-1]) + int(cap[-1]) + 64, dtype=torch.uint8, device=dev)
    t = lambda a: torch.from_numpy(a).to(dev)
    d_io, d_il, d_or = t(in_off), t(in_len.view(np.int32)), t(np.array(orders, dtype=np.int32))
    d_oo, d_oc = t(out_off), t(cap.view(np.int32))
    d_ol = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.zeros(n, dtype=torch.int32, device=dev)
    check(fn(ctx.h, d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), d_or.data_ptr(), n, d_out.data_ptr(), d_oo.data_ptr(),
             d_oc.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), *extra, stream), "encode batch")
    torch.cuda.synchronize()
    out = d_out.cpu().numpy(); ol = d_ol.cpu().numpy(); st = d_st.cpu().numpy()
    return [out[int(o):int(o) + int(l)].tobytes() if s == 0 else None for o, l, s in zip(out_off, ol, st)]


def rans4x8_encode(ctx, raws, orders, stream=0):
    """Encode byte strings with rANS 4x8 on the device (hgpu_rans4x8_encode_batch_dev)."""
    L = lib()
    L.hgpu_rans4x8_compress_bound.restype = C.c_uint32
    L.hgpu_rans4x8_compress_bound.argtypes = [C.c_uint32]
    L.hgpu_rans4x8_encode_batch_dev.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 6
    return _encode_list(ctx, L.hgpu_rans4x8_encode_batch_dev, lambda l, o: L.hgpu_rans4x8_compress_bound(l), raws, orders, stream)


def tok3_encode(ctx, blobs):
    """Encode name blocks (each a NUL/LF separated blob) with hgpu_tok3_encode_batch_host; returns [(status, bytes)]."""
    import numpy as np
    L = lib()
    L.hgpu_tok3_compress_bound.restype = C.c_uint32
    L.hgpu_tok3_compress_bound.argtypes = [C.c_uint32]
    L.hgpu_tok3_encode_batch_host.argtypes = [C.c_void_p] * 4 + [C.c_uint32] + [C.c_void_p] * 5
    n = len(blobs)
    in_len = np.array([len(c) for c in blobs], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.uint64))[:-1]]).astype(np.uint64)
    blob = np.frombuffer(b"".join(blobs) + b"\0" * 8, dtype=np.uint8)
    cap = np.array([L.hgpu_tok3_compress_bound(int(l)) for l in in_len], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum(cap.astype(np.uint64))[:-1]]).astype(np.uint64)
    out = np.zeros(int(cap.astype(np.uint64).sum()) + 8, dtype=np.uint8)
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    check(L.hgpu_tok3_encode_batch_host(ctx.h, p(blob), p(in_off), p(in_len), n, p(out), p(out_off), p(cap), p(got), p(st)),
          "tok3_encode_batch_host")
    return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]


def fqz_encode(ctx, quals, rec_lens, strat=0):
    """Encode quality blocks with fqzcomp on the device (hgpu_fqz_encode_batch_host).
    quals[i]: concatenated qualities of block i; rec_lens[i]: its record lengths.  Returns [(status, bytes)]."""
    import numpy as np
    L = lib()
    L.hgpu_fqz_compress_bound.restype = C.c_uint32
    L.hgpu_fqz_compress_bound.argtypes = [C.c_uint32, C.c_uint32]
    L.hgpu_fqz_encode_batch_host.argtypes = [C.c_void_p] * 7 + [C.c_uint32, C.c_int] + [C.c_void_p] * 5
    n = len(quals)
    in_len = np.array([len(q) for q in quals], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum(in_len.astype(np.uint64))[:-1]]).astype(np.uint64)
    blob = np.frombuffer(b"".join(quals) + b"\0" * 8, dtype=np.uint8)
    nrec = np.array([len(r) for r in rec_lens], dtype=np.uint32)
    rec_off = np.concatenate([[0], np.cumsum(nrec.astype(np.uint64))[:-1]]).astype(np.uint64)
    rec = np.array([x for r in rec_lens for x in r] + [0], dtype=np.uint32)
    cap = np.array([L.hgpu_fqz_compress_bound(int(a), int(b)) for a, b in zip(in_len, nrec)], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum((cap.astype(np.uint64) + 15) // 16 * 16)[:-1]]).astype(np.uint64)
    out = np.zeros(int(out_off[-1] + cap[-1]) + 16, dtype=np.uint8)
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    check(L.hgpu_fqz_encode_batch_host(ctx.h, p(blob), p(in_off), p(in_len), p(rec), p(rec_off), p(nrec), n, strat,
                                       p(out), p(out_off), p(cap), p(got), p(st)), "fqz_encode_batch_host")
    return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()) for i in range(n)]


def cram_parse_compression_header(payload, major=3):
    """Encoding maps of a CRAM compression-header block (uncompressed payload): (series array, description text)."""
    import numpy as np
    L = lib()
    L.hgpu_cram_parse_compression_header.restype = C.c_long
    L.hgpu_cram_parse_compression_header.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_void_p, C.c_long, C.c_char_p, C.c_size_t]
    dt = np.dtype([("key", "<u4"), ("encoding", "<i4"), ("id", "<i4", (2,))])
    arr = np.zeros(4096, dtype=dt)
    text = C.create_string_buffer(1 << 20)
    n = L.hgpu_cram_parse_compression_header(bytes(payload), len(payload), major, arr.ctypes.data, len(arr), text, len(text))
    if n < 0:
        raise HgpuError("compression header: %s" % last_error())
    return arr[:n], text.value.decode("latin-1")


def cram_scan_containers(file_np):
    """Container headers of a CRAM 3.x image: (structured array hgpu_cram_container, flat landmark array)."""
    import numpy as np
    L = lib()
    L.hgpu_cram_scan_containers.restype = C.c_long
    L.hgpu_cram_scan_containers.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_long, C.c_void_p, C.c_long]
    dt = np.dtype([("offset", "<u8"), ("data_off", "<u8"), ("record_counter", "<i8"), ("bases", "<i8"), ("length", "<i4"),
                   ("ref_id", "<i4"), ("start", "<i4"), ("span", "<i4"), ("n_records", "<i4"), ("n_blocks", "<i4"),
                   ("n_landmarks", "<i4"), ("landmark0", "<u4"), ("first_block", "<u4"), ("crc32", "<u4")])
    assert dt.itemsize == 72
    n = L.hgpu_cram_scan_containers(file_np.ctypes.data, file_np.size, None, 0, None, 0)
    if n < 0:
        raise HgpuError("CRAM container scan failed: %s" % last_error())
    arr = np.zeros(n, dtype=dt)
    L.hgpu_cram_scan_containers(file_np.ctypes.data, file_np.size, arr.ctypes.data, n, None, 0)
    nl = int(arr["n_landmarks"].sum())
    lm = np.zeros(max(1, nl), dtype=np.int32)
    L.hgpu_cram_scan_containers(file_np.ctypes.data, file_np.size, arr.ctypes.data, n, lm.ctypes.data, nl)
    return arr, lm[:nl]


def cram_parse_slice_header(payload, major=3):
    """Slice header block payload -> (dict of fields, content id list)."""
    import numpy as np
    L = lib()
    L.hgpu_cram_parse_slice_header.restype = C.c_long
    L.hgpu_cram_parse_slice_header.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_long]
    dt = np.dtype([("record_counter", "<i8"), ("ref_id", "<i4"), ("start", "<i4"), ("span", "<i4"), ("n_records", "<i4"),
                   ("n_blocks", "<i4"), ("n_content_ids", "<i4"), ("ref_base_id", "<i4"), ("md5", "u1", (16,)), ("pad", "<u4")])
    assert dt.itemsize == 56
    s = np.zeros(1, dtype=dt)
    ids = np.zeros(10000, dtype=np.int32)
    n = L.hgpu_cram_parse_slice_header(bytes(payload), len(payload), major, s.ctypes.data, ids.ctypes.data, len(ids))
    if n < 0:
        raise HgpuError("slice header: %s" % last_error())
    return s[0], ids[:n].tolist()
