"""TEST INFRASTRUCTURE -- ctypes front-end for oracle/libgen2oracle.so (the C restatement).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from gen2_uhf_rfid_reader_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libgen2oracle.so")


class OracleCfg(C.Structure):
    _fields_ = [("fs_dec", C.c_int), ("n_T1", C.c_int), ("n_PW", C.c_int), ("n_tag_bit_i", C.c_int),
                ("n_tag_bit_f", C.c_float), ("win_length", C.c_int), ("dc_length", C.c_int),
                ("len_rn16", C.c_int), ("len_epc", C.c_int), ("fixed_q", C.c_int), ("max_queries", C.c_int),
                ("max_tags", C.c_int), ("adc_rate", C.c_int), ("decim", C.c_int), ("ntaps", C.c_int),
                ("defined", C.c_int)]


def build():
    subprocess.check_call(["make", "-s", "-C", HERE, "libgen2oracle.so"])


def default_params(adc_rate=2000000, decim=5, ntaps=25, fixed_q=0, max_queries=1000, max_tags=100):
    return abi.Params(adc_rate=adc_rate, decim=decim, ntaps=ntaps, fixed_q=fixed_q, max_queries=max_queries,
                      max_tags=max_tags, device=0, reserved=0)


def derive_cfg(params=None, **kw):
    """the derived constants (OracleCfg) of a configuration, including whether it is defined; never raises"""
    if not os.path.exists(LIB):
        build()
    cfg = OracleCfg()
    C.CDLL(LIB).gen2_oracle_make_cfg(C.byref(params if params is not None else default_params(**kw)), C.byref(cfg))
    return cfg


class Oracle:
    def __init__(self, params=None, **kw):
        if not os.path.exists(LIB):
            build()
        self.lib = L = C.CDLL(LIB)
        self.params = params if params is not None else default_params(**kw)
        self.cfg = OracleCfg()
        L.gen2_oracle_make_cfg(C.byref(self.params), C.byref(self.cfg))
        if not self.cfg.defined:
            raise ValueError("adc_rate=%d, decim=%d: the reference decoder reads past the end of its windows at this "
                             "configuration, so there is no defined output to restate" % (self.params.adc_rate,
                                                                                          self.params.decim))
        L.gen2_oracle_gate.restype = C.c_int
        L.gen2_oracle_decode_decimated.restype = C.c_int
        L.gen2_oracle_decode_segments.restype = C.c_int
        L.gen2_oracle_mf.restype = C.c_size_t
        L.gen2_oracle_mf_variant.restype = C.c_size_t
        L.gen2_oracle_crc16.restype = C.c_uint16
        L.gen2_oracle_crc16_ok.restype = C.c_int
        L.gen2_oracle_cabsf.restype = C.c_float
        L.gen2_oracle_cabsf.argtypes = [C.c_float, C.c_float]

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(C.c_void_p)

    def mf(self, iq, variant=0):
        """canonical matched filter (variant 0); 1 = sequential float32, 2 = float64 accumulation"""
        raw = np.ascontiguousarray(iq, dtype=np.complex64).view(np.float32)
        n = raw.size // 2
        y = np.zeros(2 * (n // self.cfg.decim + 1), dtype=np.float32)
        ny = self.lib.gen2_oracle_mf_variant(self._p(raw), C.c_size_t(n), self.cfg.ntaps, self.cfg.decim,
                                             self._p(y), int(variant))
        return y[:2 * ny].view(np.complex64).copy()

    def gate(self, y, max_windows=4096, want_windows=False, want_avg=False):
        yy = np.ascontiguousarray(y, dtype=np.complex64).view(np.float32)
        ny = yy.size // 2
        open_idx = np.zeros(max_windows, dtype=np.int32)
        dc = np.zeros(2 * max_windows, dtype=np.float32)
        win = np.zeros(2 * max_windows * self.cfg.len_epc, dtype=np.float32) if want_windows else None
        avg = np.zeros(ny, dtype=np.float32) if want_avg else None
        n = self.lib.gen2_oracle_gate(C.byref(self.cfg), self._p(yy), C.c_size_t(ny), max_windows,
                                      self._p(open_idx), self._p(dc), self._p(win) if want_windows else None,
                                      self._p(avg) if want_avg else None)
        m = min(n, max_windows)
        out = {"n": n, "open_idx": open_idx[:m], "dc": dc[:2 * m].view(np.complex64)}
        if want_windows:
            out["windows"] = win.view(np.complex64).reshape(max_windows, self.cfg.len_epc)[:m]
        if want_avg:
            out["avg"] = avg
        return out

    def decode_window(self, kind, win):
        w = np.ascontiguousarray(win, dtype=np.complex64).view(np.float32)
        rec = np.zeros(1, dtype=abi.RESULT_DTYPE)
        self.lib.gen2_oracle_decode_window(C.byref(self.cfg), int(kind), self._p(w), w.size // 2, self._p(rec))
        return rec[0]

    def decode_decimated(self, y, max_recs=4096, segment=0):
        yy = np.ascontiguousarray(y, dtype=np.complex64).view(np.float32)
        recs = np.zeros(max_recs, dtype=abi.RESULT_DTYPE)
        n = self.lib.gen2_oracle_decode_decimated(C.byref(self.cfg), self._p(yy), C.c_size_t(yy.size // 2), segment,
                                                  self._p(recs), max_recs)
        return recs[:min(n, max_recs)], n

    def decode_segments(self, iq, segs, max_per_seg=4, want_records=True):
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        segs = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE)
        nseg = segs.size
        recs = np.zeros((nseg, max_per_seg), dtype=abi.RESULT_DTYPE) if want_records else None
        counts = np.zeros(nseg, dtype=np.int32)
        secs = C.c_double(0)
        self.lib.gen2_oracle_decode_segments(C.byref(self.cfg), self._p(raw), self._p(segs), nseg,
                                             self._p(recs) if want_records else None, max_per_seg, self._p(counts),
                                             C.byref(secs))
        return recs, counts, secs.value

    def decode_stream(self, iq, max_recs=4096):
        """one continuous raw capture -> (records, n_windows)"""
        segs = abi.make_segments([0], [np.ascontiguousarray(iq).view(np.float32).size // 2])
        recs, counts, _ = self.decode_segments(iq, segs, max_per_seg=max_recs)
        n = int(counts[0])
        return recs[0, :min(n, max_recs)], n

    def reduce_stats(self, recs, counts, continuous):
        recs = np.ascontiguousarray(recs, dtype=abi.RESULT_DTYPE)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        nseg = counts.size
        max_per = recs.size // nseg if nseg else 0
        st = abi.Stats()
        self.lib.gen2_oracle_reduce_stats(C.byref(self.cfg), self._p(recs), self._p(counts), nseg, max_per,
                                          int(bool(continuous)), C.byref(st))
        return st

    def crc16(self, data):
        b = np.frombuffer(bytes(data), dtype=np.uint8).copy()
        return int(self.lib.gen2_oracle_crc16(self._p(b), b.size))

    def crc16_ok(self, bits16):
        b = np.frombuffer(bytes(bits16), dtype=np.uint8).copy()
        return int(self.lib.gen2_oracle_crc16_ok(self._p(b)))

    def query_bits(self, q):
        out = np.zeros(22, dtype=np.uint8)
        self.lib.gen2_oracle_query_bits(int(q), self._p(out))
        return "".join(str(int(x)) for x in out)

    def cabsf(self, re, im):
        return float(self.lib.gen2_oracle_cabsf(C.c_float(re), C.c_float(im)))
