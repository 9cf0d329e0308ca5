"""ctypes binding of librfid_b200.so (include/rfid_b200.h) + a thin, torch-aware wrapper.

PyTorch is used only for device memory, streams and (elsewhere) torch.distributed; every
signal-path operation goes through the C-ABI into the hand-written sm_90a kernels.  There is no
CPU fallback: constructing `Gen2Rx` without the compiled library or without an H100 raises.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .build import LIB, build_library

_lib = None


class RfidB200Error(RuntimeError):
    pass


def load_library():
    """dlopen the in-tree library (building it first if the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    path = LIB
    override = os.environ.get("RFID_B200_LIB")   # developer aid: a library built with other flags (tools/variants.sh)
    if override:
        path = override
    else:
        try:
            path = build_library()
        except Exception:
            if not os.path.exists(LIB):
                raise
    if not os.path.exists(path):
        raise RfidB200Error("librfid_b200.so is missing: run `python -m gen2_uhf_rfid_reader_b200.build` "
                            "(there is no CPU fallback)")
    L = C.CDLL(path)
    vp, ip, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float)
    L.rfid_b200_abi_version.restype = C.c_int
    L.rfid_b200_strerror.restype = C.c_char_p
    L.rfid_b200_strerror.argtypes = [C.c_int]
    L.rfid_b200_last_cuda_error.restype = C.c_char_p
    L.rfid_b200_last_cuda_error.argtypes = [vp]
    L.rfid_b200_default_params.argtypes = [C.POINTER(abi.Params)]
    L.rfid_b200_create.restype = C.c_int
    L.rfid_b200_create.argtypes = [C.POINTER(abi.Params), C.POINTER(vp)]
    L.rfid_b200_destroy.argtypes = [vp]
    L.rfid_b200_window_length.restype = C.c_int
    L.rfid_b200_window_length.argtypes = [vp, C.c_int]
    L.rfid_b200_fs_dec.restype = C.c_int
    L.rfid_b200_fs_dec.argtypes = [vp]
    L.rfid_b200_decode_capture.restype = C.c_int
    L.rfid_b200_decode_capture.argtypes = [vp, vp, C.c_size_t, vp, C.c_int, C.c_int, vp, vp, vp]
    L.rfid_b200_decode_capture_host.restype = C.c_int
    L.rfid_b200_decode_capture_host.argtypes = [vp, vp, C.c_size_t, vp, C.c_int, C.c_int, vp, vp]
    L.rfid_b200_last_launch_count.restype = C.c_int
    L.rfid_b200_last_launch_count.argtypes = [vp]
    L.rfid_b200_kernel_time.restype = C.c_int
    L.rfid_b200_kernel_time.argtypes = [vp, C.c_int, fp, ip]
    L.rfid_b200_enable_kernel_timing.restype = C.c_int
    L.rfid_b200_enable_kernel_timing.argtypes = [vp, C.c_int]
    L.rfid_b200_set_window_tap.restype = C.c_int
    L.rfid_b200_set_window_tap.argtypes = [vp, vp]
    L.rfid_b200_reduce_stats.restype = C.c_int
    L.rfid_b200_reduce_stats.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.Stats)]
    L.rfid_b200_gate_work.restype = C.c_int
    L.rfid_b200_gate_work.argtypes = [vp, C.c_int, vp, C.c_int, vp, C.c_int, ip, ip, ip, vp]
    L.rfid_b200_decoder_work.restype = C.c_int
    L.rfid_b200_decoder_work.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]
    L.rfid_b200_mf_work.restype = C.c_int
    L.rfid_b200_mf_work.argtypes = [vp, vp, C.c_int, vp, C.c_int, ip]
    L.rfid_b200_default_segmenter.argtypes = [C.POINTER(abi.Segmenter)]
    L.rfid_b200_segment_capture.restype = C.c_int
    L.rfid_b200_segment_capture.argtypes = [vp, vp, C.c_size_t, C.POINTER(abi.Segmenter), vp, C.c_int, ip, vp]
    L.rfid_b200_ingest_capture_host.restype = C.c_int
    L.rfid_b200_ingest_capture_host.argtypes = [vp, vp, C.c_size_t, C.POINTER(abi.Segmenter), C.c_int, vp, C.c_int, ip,
                                                vp, vp]
    L.rfid_b200_tx_synth.restype = C.c_int
    L.rfid_b200_tx_synth.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_size_t, C.POINTER(C.c_size_t), vp]
    L.rfid_b200_default_sim.argtypes = [C.POINTER(abi.SimParams)]
    L.rfid_b200_sim_segment_length.restype = C.c_int
    L.rfid_b200_sim_segment_length.argtypes = [vp, C.POINTER(abi.SimParams)]
    L.rfid_b200_sim_capture.restype = C.c_int
    L.rfid_b200_sim_capture.argtypes = [vp, C.POINTER(abi.SimParams), C.c_int64, C.c_int, vp, vp, vp, vp]
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "rfid_b200_abi_version", "rfid_b200_strerror", "rfid_b200_last_cuda_error", "rfid_b200_default_params",
    "rfid_b200_create", "rfid_b200_destroy", "rfid_b200_window_length", "rfid_b200_fs_dec",
    "rfid_b200_decode_capture", "rfid_b200_decode_capture_host", "rfid_b200_last_launch_count",
    "rfid_b200_kernel_time", "rfid_b200_enable_kernel_timing", "rfid_b200_set_window_tap",
    "rfid_b200_reduce_stats", "rfid_b200_gate_work", "rfid_b200_decoder_work", "rfid_b200_mf_work",
    "rfid_b200_default_segmenter", "rfid_b200_segment_capture", "rfid_b200_ingest_capture_host",
    "rfid_b200_tx_synth", "rfid_b200_default_sim", "rfid_b200_sim_segment_length", "rfid_b200_sim_capture",
]


def default_sim(**kw):
    p = abi.SimParams()
    load_library().rfid_b200_default_sim(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, type(getattr(p, k))(v))
    return p


def default_segmenter(**kw):
    sp = abi.Segmenter()
    load_library().rfid_b200_default_segmenter(C.byref(sp))
    for k, v in kw.items():
        setattr(sp, k, type(getattr(sp, k))(v))
    return sp


def default_params(**kw):
    p = abi.Params()
    load_library().rfid_b200_default_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, int(v))
    return p


class Gen2Rx:
    """One receive-chain context (capture mode and block mode)."""

    def __init__(self, params=None, **kw):
        self.lib = load_library()
        self.params = params if params is not None else default_params(**kw)
        h = C.c_void_p()
        rc = self.lib.rfid_b200_create(C.byref(self.params), C.byref(h))
        if rc == abi.EINVAL:
            raise RfidB200Error("rfid_b200_create: %s: the parameters are out of range, or the configuration is not well "
                                "defined (at adc_rate=%d, decim=%d the reference decoder reads past the end of its windows; "
                                "see rfid_b200.h)" % (self.lib.rfid_b200_strerror(rc).decode(), self.params.adc_rate,
                                                      self.params.decim))
        if rc != 0:
            raise RfidB200Error("rfid_b200_create: %s" % self.lib.rfid_b200_strerror(rc).decode())
        self.h = h
        self.len_rn16 = self.lib.rfid_b200_window_length(h, abi.RN16)
        self.len_epc = self.lib.rfid_b200_window_length(h, abi.EPC)
        self.fs_dec = self.lib.rfid_b200_fs_dec(h)

    def close(self):
        if getattr(self, "h", None):
            self.lib.rfid_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc, what):
        if rc != 0:
            raise RfidB200Error("%s: %s (%s)" % (what, self.lib.rfid_b200_strerror(rc).decode(),
                                                 self.lib.rfid_b200_last_cuda_error(self.h).decode()))

    # ---------------------------------------------------------------- capture mode
    def decode_capture(self, iq, segs, max_windows=4, results=None, counts=None, stream=None):
        """iq: CUDA complex64 (or float32 interleaved) tensor; segs: CUDA uint8/int64 tensor holding
        rfid_b200_segment[nseg] (see `segments_to_device`).  Asynchronous on `stream` (default: the
        current torch stream).  Returns (results uint8[nseg*max_windows,64], counts int32[nseg])."""
        import torch
        nseg = segs.numel() * segs.element_size() // 16
        n_raw = iq.numel() if iq.is_complex() else iq.numel() // 2
        if results is None:
            results = torch.zeros((nseg * max_windows, 64), dtype=torch.uint8, device=iq.device)
        if counts is None:
            counts = torch.zeros(nseg, dtype=torch.int32, device=iq.device)
        s = stream if stream is not None else torch.cuda.current_stream(iq.device)
        rc = self.lib.rfid_b200_decode_capture(self.h, iq.data_ptr(), n_raw, segs.data_ptr(), nseg, max_windows,
                                               results.data_ptr(), counts.data_ptr(), s.cuda_stream)
        self._ck(rc, "rfid_b200_decode_capture")
        return results, counts

    def decode_capture_host(self, iq, segs, max_windows=4):
        """Host arrays in, host records out (copies inside): iq complex64 ndarray, segs SEGMENT_DTYPE."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        segs = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE)
        nseg = segs.size
        recs = np.zeros((nseg, max_windows), dtype=abi.RESULT_DTYPE)
        counts = np.zeros(nseg, dtype=np.int32)
        rc = self.lib.rfid_b200_decode_capture_host(self.h, raw.ctypes.data, raw.size // 2, segs.ctypes.data, nseg,
                                                    max_windows, recs.ctypes.data, counts.ctypes.data)
        self._ck(rc, "rfid_b200_decode_capture_host")
        return recs, counts

    def decode_capture_host_ptr(self, iq_ptr, n_raw, segs_ptr, nseg, max_windows, res_ptr, cnt_ptr):
        """Same call on raw (e.g. pinned) host pointers: no Python-side copies."""
        rc = self.lib.rfid_b200_decode_capture_host(self.h, iq_ptr, n_raw, segs_ptr, nseg, max_windows, res_ptr, cnt_ptr)
        self._ck(rc, "rfid_b200_decode_capture_host")

    # ---------------------------------------------------------------- capture ingest
    def segment_capture(self, iq, segmenter=None, capacity=None, stream=None):
        """CW-gap segment table (SEGMENT_DTYPE ndarray) of a CUDA capture tensor."""
        import torch
        n_raw = iq.numel() if iq.is_complex() else iq.numel() // 2
        cap = int(capacity) if capacity is not None else max(16, n_raw // 4096)
        segs = np.zeros(cap, dtype=abi.SEGMENT_DTYPE)
        n = C.c_int(0)
        s = stream if stream is not None else torch.cuda.current_stream(iq.device)
        rc = self.lib.rfid_b200_segment_capture(self.h, iq.data_ptr(), n_raw, C.byref(segmenter) if segmenter else None,
                                                segs.ctypes.data, cap, C.byref(n), s.cuda_stream)
        self._ck(rc, "rfid_b200_segment_capture")
        return segs[:n.value].copy()

    def ingest_capture_host(self, iq, segmenter=None, max_windows=4, capacity=None):
        """Recorded capture (host complex64 ndarray, e.g. np.fromfile/np.memmap) -> (segs, records, counts)."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        n_raw = raw.size // 2
        cap = int(capacity) if capacity is not None else max(16, n_raw // 4096)
        segs = np.zeros(cap, dtype=abi.SEGMENT_DTYPE)
        recs = np.zeros((cap, max_windows), dtype=abi.RESULT_DTYPE)
        counts = np.zeros(cap, dtype=np.int32)
        n = C.c_int(0)
        rc = self.lib.rfid_b200_ingest_capture_host(self.h, raw.ctypes.data, n_raw, C.byref(segmenter) if segmenter else None,
                                                    max_windows, segs.ctypes.data, cap, C.byref(n), recs.ctypes.data,
                                                    counts.ctypes.data)
        self._ck(rc, "rfid_b200_ingest_capture_host")
        k = n.value
        return segs[:k].copy(), recs[:k].copy(), counts[:k].copy()

    # ---------------------------------------------------------------- TX synthesiser / slot simulator
    def tx_synth(self, script, dac_rate=1000000, device="cuda:0"):
        """script: iterable of (kind, arg) -> float32 CUDA tensor with the reader's TX envelope."""
        import torch
        scr = np.array([(int(k), int(a)) for k, a in script], dtype=abi.TX_COMMAND_DTYPE)
        n = C.c_size_t(0)
        self._ck(self.lib.rfid_b200_tx_synth(self.h, scr.ctypes.data, scr.size, dac_rate, None, 0, C.byref(n), None),
                 "rfid_b200_tx_synth")
        out = torch.empty(n.value, dtype=torch.float32, device=device)
        s = torch.cuda.current_stream(out.device)
        self._ck(self.lib.rfid_b200_tx_synth(self.h, scr.ctypes.data, scr.size, dac_rate, out.data_ptr(), out.numel(),
                                             C.byref(n), s.cuda_stream), "rfid_b200_tx_synth")
        return out

    def sim_segment_length(self, sim):
        n = self.lib.rfid_b200_sim_segment_length(self.h, C.byref(sim))
        if n < 0:
            self._ck(n, "rfid_b200_sim_segment_length")
        return n

    def sim_capture(self, sim, nseg, first_segment=0, device="cuda:0", out=None):
        """Generate `nseg` inventory slots on the GPU.  Returns dict(iq complex64 CUDA tensor, segs CUDA uint8
        tensor holding rfid_b200_segment[nseg], truth CUDA uint8 tensor [nseg,48] (abi.SIM_TRUTH_DTYPE))."""
        import torch
        seg_len = self.sim_segment_length(sim)
        dev = torch.device(device)
        iq = out if out is not None else torch.empty(nseg * seg_len, dtype=torch.complex64, device=dev)
        segs = torch.zeros((nseg, 16), dtype=torch.uint8, device=dev)
        truth = torch.zeros((nseg, 48), dtype=torch.uint8, device=dev)
        s = torch.cuda.current_stream(dev)
        self._ck(self.lib.rfid_b200_sim_capture(self.h, C.byref(sim), first_segment, nseg, iq.data_ptr(), segs.data_ptr(),
                                                truth.data_ptr(), s.cuda_stream), "rfid_b200_sim_capture")
        return {"iq": iq, "segs": segs, "truth": truth, "segment_len": seg_len}

    def set_window_tap(self, tensor_or_none):
        ptr = tensor_or_none.data_ptr() if tensor_or_none is not None else None
        self._ck(self.lib.rfid_b200_set_window_tap(self.h, ptr), "rfid_b200_set_window_tap")

    def enable_kernel_timing(self, on=True):
        self._ck(self.lib.rfid_b200_enable_kernel_timing(self.h, int(on)), "rfid_b200_enable_kernel_timing")

    def kernel_time(self, reset=True):
        ms, n = C.c_float(0), C.c_int(0)
        self._ck(self.lib.rfid_b200_kernel_time(self.h, int(reset), C.byref(ms), C.byref(n)), "rfid_b200_kernel_time")
        return ms.value, n.value

    def last_launch_count(self):
        return self.lib.rfid_b200_last_launch_count(self.h)

    def reduce_stats(self, recs, counts, continuous):
        recs = np.ascontiguousarray(recs, dtype=abi.RESULT_DTYPE)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        nseg = counts.size
        max_per = recs.size // nseg if nseg else 1
        st = abi.Stats()
        self._ck(self.lib.rfid_b200_reduce_stats(self.h, recs.ctypes.data, counts.ctypes.data, nseg, max(1, max_per),
                                                 int(bool(continuous)), C.byref(st)), "rfid_b200_reduce_stats")
        return st

    # ---------------------------------------------------------------- block mode
    def gate_work(self, chunk, seek=0, want_magn2=False):
        x = np.ascontiguousarray(chunk, dtype=np.complex64)
        n = x.size
        out = np.zeros(max(n, 1), dtype=np.complex64)
        m2 = np.zeros(max(n, 1), dtype=np.float32) if want_magn2 else None
        c, w, cl = C.c_int(0), C.c_int(0), C.c_int(0)
        rc = self.lib.rfid_b200_gate_work(self.h, int(seek), x.ctypes.data, n, out.ctypes.data, max(n, 1),
                                          C.byref(c), C.byref(w), C.byref(cl), m2.ctypes.data if want_magn2 else None)
        self._ck(rc, "rfid_b200_gate_work")
        res = {"consumed": c.value, "written": w.value, "closed": cl.value, "out": out[:w.value]}
        if want_magn2:
            res["magn2"] = m2[:w.value]
        return res

    def decoder_work(self, kind, window):
        w = np.ascontiguousarray(window, dtype=np.complex64)
        rec = np.zeros(1, dtype=abi.RESULT_DTYPE)
        bits = np.zeros(128, dtype=np.float32)
        rc = self.lib.rfid_b200_decoder_work(self.h, int(kind), w.ctypes.data, w.size, rec.ctypes.data, bits.ctypes.data)
        self._ck(rc, "rfid_b200_decoder_work")
        return rec[0], bits[:16 if kind == abi.RN16 else 128]

    def mf_work(self, chunk):
        x = np.ascontiguousarray(chunk, dtype=np.complex64)
        cap = x.size // self.params.decim + 2
        out = np.zeros(cap, dtype=np.complex64)
        w = C.c_int(0)
        rc = self.lib.rfid_b200_mf_work(self.h, x.ctypes.data, x.size, out.ctypes.data, cap, C.byref(w))
        self._ck(rc, "rfid_b200_mf_work")
        return out[:w.value]


def segments_to_device(segs, device):
    """SEGMENT_DTYPE ndarray -> CUDA uint8 tensor holding the same bytes."""
    import torch
    b = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE).view(np.uint8)
    return torch.from_numpy(b.copy()).to(device)


def results_to_numpy(results, counts, max_windows):
    """device uint8[nseg*max_windows,64] + int32[nseg] -> (RESULT_DTYPE[nseg,max_windows], int32[nseg])"""
    r = results.cpu().numpy().reshape(-1).view(abi.RESULT_DTYPE)
    c = counts.cpu().numpy()
    return r.reshape(c.size, max_windows), c
