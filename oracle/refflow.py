"""TEST INFRASTRUCTURE -- ctypes front-end for the flow-driver libraries.

`RefFlow` loads oracle/_ref/libgen2ref[_q4].so (the reference's own blocks,
compiled unchanged by oracle/build_ref.sh + oracle/flow_driver.cc) and exposes
stream / segment decoding that returns `rfid_b200_window_result` records.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this module.  The product never does.
"""
import ctypes as C
import os

import numpy as np

from gen2_uhf_rfid_reader_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))


def ref_lib_path(fixed_q=0):
    name = "libgen2ref.so" if fixed_q == 0 else "libgen2ref_q%d.so" % fixed_q
    return os.path.join(HERE, "_ref", name)


def ref_available(fixed_q=0):
    return os.path.exists(ref_lib_path(fixed_q))


class FlowLib:
    """A flow-driver shared object (reference blocks or this repo's host blocks)."""

    def __init__(self, path):
        self.path = path
        self.lib = C.CDLL(path)
        L = self.lib
        f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        L.gen2flow_run_stream.restype = C.c_int
        L.gen2flow_run_stream.argtypes = [f32p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_int, C.POINTER(abi.Stats), C.c_char_p, C.c_size_t,
                                          f32p, C.c_size_t, C.POINTER(C.c_size_t), f32p]
        L.gen2flow_run_decimated.restype = C.c_int
        L.gen2flow_run_decimated.argtypes = [f32p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                             C.POINTER(abi.Stats)]
        L.gen2flow_run_segments.restype = C.c_int
        L.gen2flow_run_segments.argtypes = [f32p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p, C.c_int, i32p, C.POINTER(C.c_double)]
        L.gen2flow_reader_script.restype = C.c_int
        L.gen2flow_reader_script.argtypes = [f32p, C.c_int, C.c_int, f32p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.gen2flow_is_reference.restype = C.c_int
        L.gen2flow_fixed_q.restype = C.c_int
        L.gen2flow_set_logging.argtypes = [C.c_int, C.c_int]

    @property
    def is_reference(self):
        return bool(self.lib.gen2flow_is_reference())

    @property
    def fixed_q(self):
        return int(self.lib.gen2flow_fixed_q())

    @staticmethod
    def _f32(a):
        a = np.ascontiguousarray(a, dtype=np.float32)
        return a, a.ctypes.data_as(C.POINTER(C.c_float))

    def run_stream(self, iq, adc_rate=2000000, decim=5, ntaps=25, dac_rate=1000000, chunk=4096,
                   max_recs=4096, want_tx=False, want_y=False):
        """iq: complex64 (or interleaved float32) raw capture, decoded as ONE continuous stream.
        Returns dict(records, stats, text[, tx][, y])."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        raw, p = self._f32(raw)
        n_raw = raw.size // 2
        recs = np.zeros(max_recs, dtype=abi.RESULT_DTYPE)
        stats = abi.Stats()
        text = C.create_string_buffer(4096)
        tx = np.zeros(8_000_000 if want_tx else 1, dtype=np.float32)
        tx_n = C.c_size_t(0)
        y = np.zeros(2 * (n_raw // decim + 1) if want_y else 2, dtype=np.float32)
        n = self.lib.gen2flow_run_stream(p, n_raw, adc_rate, decim, ntaps, dac_rate, chunk,
                                         recs.ctypes.data, max_recs, C.byref(stats), text, len(text),
                                         tx.ctypes.data_as(C.POINTER(C.c_float)) if want_tx else None, tx.size,
                                         C.byref(tx_n), y.ctypes.data_as(C.POINTER(C.c_float)) if want_y else None)
        if n < 0:
            raise RuntimeError("gen2flow_run_stream failed: %d" % n)
        out = {"records": recs[:min(n, max_recs)], "n_windows": n, "stats": stats, "text": text.value.decode()}
        if want_tx:
            out["tx"] = tx[:tx_n.value].copy()
        if want_y:
            out["y"] = y[:2 * (n_raw // decim)].view(np.complex64).copy()
        return out

    def reader_script(self, rn16_bits, dac_rate=1000000):
        """scripted run of the reader block alone (CPU only): returns (tx envelope, n_queries_sent)"""
        bits = np.ascontiguousarray(rn16_bits, dtype=np.float32).reshape(-1, 16)
        tx = np.zeros((bits.shape[0] * 12000 + 8000) * max(1, -(-dac_rate // 1000000)), dtype=np.float32)
        n = C.c_size_t(0)
        nq = self.lib.gen2flow_reader_script(bits.ctypes.data_as(C.POINTER(C.c_float)), bits.shape[0], dac_rate,
                                             tx.ctypes.data_as(C.POINTER(C.c_float)), tx.size, C.byref(n))
        return tx[:n.value].copy(), nq

    def run_decimated(self, y, fs_dec=400000, dac_rate=1000000, chunk=4096, max_recs=4096):
        yy = np.ascontiguousarray(y, dtype=np.complex64).view(np.float32)
        yy, p = self._f32(yy)
        recs = np.zeros(max_recs, dtype=abi.RESULT_DTYPE)
        stats = abi.Stats()
        n = self.lib.gen2flow_run_decimated(p, yy.size // 2, fs_dec, dac_rate, chunk, recs.ctypes.data, max_recs,
                                            C.byref(stats))
        if n < 0:
            raise RuntimeError("gen2flow_run_decimated failed: %d" % n)
        return {"records": recs[:min(n, max_recs)], "n_windows": n, "stats": stats}

    def run_segments(self, iq, segs, adc_rate=2000000, decim=5, ntaps=25, dac_rate=1000000, chunk=4096,
                     max_per_seg=4, want_records=True):
        """Independent segments, fresh blocks each.  Returns (records[nseg,max_per_seg], counts[nseg], seconds)."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        raw, p = self._f32(raw)
        segs = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE)
        nseg = segs.size
        recs = np.zeros((nseg, max_per_seg), dtype=abi.RESULT_DTYPE) if want_records else None
        counts = np.zeros(nseg, dtype=np.int32)
        secs = C.c_double(0.0)
        rc = self.lib.gen2flow_run_segments(p, segs.ctypes.data, nseg, adc_rate, decim, ntaps, dac_rate, chunk,
                                            recs.ctypes.data if want_records else None, max_per_seg,
                                            counts.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(secs))
        if rc < 0:
            raise RuntimeError("gen2flow_run_segments failed: %d" % rc)
        return recs, counts, secs.value


def B200Flow():
    """the A/B harness around THIS repo's host blocks (needs an H100 at run time)"""
    path = os.path.join(HERE, "libgen2flow_b200.so")
    if not os.path.exists(path):
        raise FileNotFoundError(path + " (make -C oracle flow_b200)")
    return FlowLib(path)


def RefFlow(fixed_q=0):
    path = ref_lib_path(fixed_q)
    if not os.path.exists(path):
        raise FileNotFoundError(path + " (run oracle/build_ref.sh where /root/reference exists)")
    return FlowLib(path)
