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

# Default int16 -> float factor of sc16 captures: 1/32767, the factor UHD's host converters conventionally apply when they
# widen the radio's sc16 samples to fc32 (full scale +-32767 -> +-1.0).  Decoding never depends on the value: an sc16
# capture decodes, bit for bit, like its fc32 conversion np.float32(i) * np.float32(scale) with the same float.
SC16_SCALE = float(np.float32(1.0 / 32767.0))


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
    for name, (restype, argtypes) in _SIGNATURES.items():
        f = getattr(L, name)
        f.restype, f.argtypes = restype, argtypes
    _lib = L
    return L


_vp, _int, _size, _float = C.c_void_p, C.c_int, C.c_size_t, C.c_float
_ip, _P = C.POINTER(C.c_int), C.POINTER
# Every function include/rfid_b200.h declares: name -> (restype, argtypes).  The void functions keep ctypes' default
# restype, c_int.
_SIGNATURES = {
    "rfid_b200_abi_version": (_int, []),
    "rfid_b200_strerror": (C.c_char_p, [_int]),
    "rfid_b200_last_cuda_error": (C.c_char_p, [_vp]),
    "rfid_b200_default_params": (_int, [_P(abi.Params)]),
    "rfid_b200_create": (_int, [_P(abi.Params), _P(_vp)]),
    "rfid_b200_destroy": (_int, [_vp]),
    "rfid_b200_window_length": (_int, [_vp, _int]),
    "rfid_b200_fs_dec": (_int, [_vp]),
    "rfid_b200_decode_capture": (_int, [_vp, _vp, _size, _vp, _int, _int, _vp, _vp, _vp]),
    "rfid_b200_decode_capture_sc16": (_int, [_vp, _vp, _size, _float, _vp, _int, _int, _vp, _vp, _vp]),
    "rfid_b200_decode_capture_host": (_int, [_vp, _vp, _size, _vp, _int, _int, _vp, _vp]),
    "rfid_b200_last_launch_count": (_int, [_vp]),
    "rfid_b200_kernel_time": (_int, [_vp, _int, _P(_float), _ip]),
    "rfid_b200_enable_kernel_timing": (_int, [_vp, _int]),
    "rfid_b200_set_window_tap": (_int, [_vp, _vp]),
    "rfid_b200_reduce_stats": (_int, [_vp, _vp, _vp, _int, _int, _int, _P(abi.Stats)]),
    "rfid_b200_gate_work": (_int, [_vp, _int, _vp, _int, _vp, _int, _ip, _ip, _ip, _vp]),
    "rfid_b200_decoder_work": (_int, [_vp, _int, _vp, _int, _vp, _vp]),
    "rfid_b200_mf_work": (_int, [_vp, _vp, _int, _vp, _int, _ip]),
    "rfid_b200_default_segmenter": (_int, [_P(abi.Segmenter)]),
    "rfid_b200_segment_capture": (_int, [_vp, _vp, _size, _P(abi.Segmenter), _vp, _int, _ip, _vp]),
    "rfid_b200_segment_capture_sc16": (_int, [_vp, _vp, _size, _float, _P(abi.Segmenter), _vp, _int, _ip, _vp]),
    "rfid_b200_ingest_capture_host": (_int, [_vp, _vp, _size, _P(abi.Segmenter), _int, _vp, _int, _ip, _vp, _vp]),
    "rfid_b200_ingest_capture_host_sc16": (_int, [_vp, _vp, _size, _float, _P(abi.Segmenter), _int, _vp, _int, _ip, _vp,
                                                  _vp]),
    "rfid_b200_tx_synth": (_int, [_vp, _vp, _int, _int, _vp, _size, _P(_size), _vp]),
    "rfid_b200_default_sim": (_int, [_P(abi.SimParams)]),
    "rfid_b200_sim_segment_length": (_int, [_vp, _P(abi.SimParams)]),
    "rfid_b200_sim_capture": (_int, [_vp, _P(abi.SimParams), C.c_int64, _int, _vp, _vp, _vp, _vp]),
    "rfid_b200_default_cmd_params": (_int, [_P(abi.CmdParams)]),
    "rfid_b200_decode_commands": (_int, [_vp, _vp, _size, _vp, _int, _P(abi.CmdParams), _int, _vp, _vp, _vp]),
    "rfid_b200_decode_commands_sc16": (_int, [_vp, _vp, _size, _float, _vp, _int, _P(abi.CmdParams), _int, _vp, _vp,
                                              _vp]),
    "rfid_b200_decode_commands_host": (_int, [_vp, _vp, _size, _vp, _int, _P(abi.CmdParams), _int, _vp, _vp]),
    "rfid_b200_default_quality_params": (_int, [_P(abi.QualityParams)]),
    "rfid_b200_window_quality": (_int, [_vp, _vp, _vp, _vp, _int, _int, _P(abi.QualityParams), _vp, _vp]),
    "rfid_b200_default_recover_params": (_int, [_P(abi.RecoverParams)]),
    "rfid_b200_recover_epc": (_int, [_vp, _vp, _vp, _vp, _vp, _int, _int, _P(abi.RecoverParams), _vp, _vp]),
    "rfid_b200_default_report_params": (_int, [_P(abi.ReportParams)]),
    "rfid_b200_tag_report": (_int, [_vp, _vp, _vp, _vp, _int, _int, _vp, _vp, _P(abi.ReportParams), _int, _vp, _vp, _vp,
                                    _vp]),
    "rfid_b200_default_match_params": (_int, [_P(abi.MatchParams)]),
    "rfid_b200_match_epc": (_int, [_vp, _vp, _vp, _vp, _vp, _int, _int, _vp, _vp, _int, _P(abi.MatchParams), _vp, _vp,
                                   _vp]),
}
EXPORTED_SYMBOLS = list(_SIGNATURES)


def _capture(iq, scale):
    """(entry-point suffix, leading arguments) of a CUDA capture: ("", (pointer, samples)) for complex64 or float32
    interleaved (fc32), ("_sc16", (pointer, samples, scale)) for a torch.int16 tensor shaped (2n,) or (n, 2) holding
    interleaved I, Q (UHD's sc16)"""
    import torch
    if iq.dtype != torch.int16:
        return "", (iq.data_ptr(), iq.numel() if iq.is_complex() else iq.numel() // 2)
    if iq.dim() == 2 and iq.shape[1] != 2 or iq.dim() > 2 or iq.numel() % 2:
        raise ValueError("an int16 capture is shaped (2n,) or (n, 2): interleaved I, Q")
    if not iq.is_contiguous():
        raise ValueError("an int16 capture must be contiguous")
    return "_sc16", (iq.data_ptr(), iq.numel() // 2, scale)


def _stream(stream, device):
    """the CUDA handle of `stream`, or of the current torch stream on `device`"""
    import torch
    return (stream if stream is not None else torch.cuda.current_stream(device)).cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _ref(params):
    return C.byref(params) if params is not None else None


def _defaults(struct, fill, kw, cast=None):
    """`struct` filled by the library's `fill`, then the fields in kw set (converted by cast, by default to the
    field's type)"""
    p = struct()
    getattr(load_library(), fill)(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, (cast or type(getattr(p, k)))(v))
    return p


def default_sim(**kw):
    return _defaults(abi.SimParams, "rfid_b200_default_sim", kw)


def default_segmenter(**kw):
    return _defaults(abi.Segmenter, "rfid_b200_default_segmenter", kw)


def default_cmd_params(**kw):
    """rfid_b200_cmd_params with the library's defaults (level_frac 0.5, level_abs 0, gap_us 400), fields set by kw."""
    return _defaults(abi.CmdParams, "rfid_b200_default_cmd_params", kw)


def default_quality_params(**kw):
    """rfid_b200_quality_params with the library's defaults (empty_db 9.5, single_snr_db 8.8), fields set by kw."""
    return _defaults(abi.QualityParams, "rfid_b200_default_quality_params", kw)


def default_recover_params(**kw):
    """rfid_b200_recover_params with the library's defaults (positions 12, max_flips 4, min_snr_db 7.0), fields set by
    kw."""
    return _defaults(abi.RecoverParams, "rfid_b200_default_recover_params", kw)


def default_report_params(**kw):
    """rfid_b200_report_params with the library's defaults (check_length 1), fields set by kw."""
    return _defaults(abi.ReportParams, "rfid_b200_default_report_params", kw)


def default_match_params(**kw):
    """rfid_b200_match_params with the library's defaults (max_cost 12, min_margin 4), fields set by kw."""
    return _defaults(abi.MatchParams, "rfid_b200_default_match_params", kw)


def default_params(**kw):
    return _defaults(abi.Params, "rfid_b200_default_params", kw, int)


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

    def _call(self, name, *args):
        """lib.name(context, *args), raising on an error code"""
        self._ck(getattr(self.lib, name)(self.h, *args), name)

    def _check_tap(self, windows, nseg, max_windows):
        if windows.numel() * windows.element_size() < nseg * max_windows * self.len_epc * 8:
            raise ValueError("the window tap holds fewer than nseg * max_windows * len_epc complex samples")

    # ---------------------------------------------------------------- capture mode
    def decode_capture(self, iq, segs, max_windows=4, results=None, counts=None, stream=None, scale=SC16_SCALE):
        """iq: CUDA complex64 (or float32 interleaved) tensor, or a torch.int16 tensor shaped (2n,) or (n, 2) holding an
        sc16 capture (interleaved int16 I, Q), decoded as its conversion I * scale, Q * scale (`SC16_SCALE` by default);
        segs: CUDA uint8/int64 tensor holding rfid_b200_segment[nseg] (see `segments_to_device`).  Asynchronous on
        `stream` (default: the current torch stream).  Returns (results uint8[nseg*max_windows,64], counts int32[nseg])."""
        import torch
        nseg = segs.numel() * segs.element_size() // 16
        fmt, cap = _capture(iq, scale)
        if results is None:
            results = torch.zeros((nseg * max_windows, 64), dtype=torch.uint8, device=iq.device)
        if counts is None:
            counts = torch.zeros(nseg, dtype=torch.int32, device=iq.device)
        self._call("rfid_b200_decode_capture" + fmt, *cap, segs.data_ptr(), nseg, max_windows, results.data_ptr(),
                   counts.data_ptr(), _stream(stream, iq.device))
        return results, counts

    def decode_capture_host(self, iq, segs, max_windows=4):
        """Host arrays in, host records out (copies inside): iq complex64 ndarray, segs SEGMENT_DTYPE."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        segs = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE)
        nseg = segs.size
        recs = np.zeros((nseg, max_windows), dtype=abi.RESULT_DTYPE)
        counts = np.zeros(nseg, dtype=np.int32)
        self._call("rfid_b200_decode_capture_host", raw.ctypes.data, raw.size // 2, segs.ctypes.data, nseg, max_windows,
                   recs.ctypes.data, counts.ctypes.data)
        return recs, counts

    def decode_capture_host_ptr(self, iq_ptr, n_raw, segs_ptr, nseg, max_windows, res_ptr, cnt_ptr):
        """Same call on raw (e.g. pinned) host pointers: no Python-side copies."""
        self._call("rfid_b200_decode_capture_host", iq_ptr, n_raw, segs_ptr, nseg, max_windows, res_ptr, cnt_ptr)

    # ---------------------------------------------------------------- capture mode: the reader's commands
    def decode_commands(self, iq, segs, max_commands=8, commands=None, counts=None, stream=None, scale=SC16_SCALE,
                        params=None):
        """The reader's PIE commands in every segment (rule: include/rfid_b200.h).  iq and segs as in `decode_capture`
        (complex64 / float32 interleaved, or an sc16 torch.int16 tensor decoded as its conversion); params: `CmdParams`
        (None: defaults, see `default_cmd_params`).  Asynchronous on `stream`.  Returns (commands uint8[nseg*max,64],
        counts int32[nseg]); `commands_to_numpy` views them as COMMAND_DTYPE."""
        import torch
        nseg = segs.numel() * segs.element_size() // 16
        fmt, cap = _capture(iq, scale)
        if commands is None:
            commands = torch.zeros((nseg * max_commands, 64), dtype=torch.uint8, device=iq.device)
        if counts is None:
            counts = torch.zeros(nseg, dtype=torch.int32, device=iq.device)
        self._call("rfid_b200_decode_commands" + fmt, *cap, segs.data_ptr(), nseg, _ref(params), max_commands,
                   commands.data_ptr(), counts.data_ptr(), _stream(stream, iq.device))
        return commands, counts

    def decode_commands_host(self, iq, segs, max_commands=8, params=None):
        """Host arrays in, host records out: iq complex64 ndarray, segs SEGMENT_DTYPE -> (COMMAND_DTYPE[nseg, max],
        int32[nseg])."""
        raw = np.ascontiguousarray(iq).view(np.float32).ravel()
        segs = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE)
        nseg = segs.size
        cmds = np.zeros((nseg, max_commands), dtype=abi.COMMAND_DTYPE)
        counts = np.zeros(nseg, dtype=np.int32)
        self._call("rfid_b200_decode_commands_host", raw.ctypes.data, raw.size // 2, segs.ctypes.data, nseg,
                   _ref(params), max_commands, cmds.ctypes.data if cmds.size else None, counts.ctypes.data)
        return cmds, counts

    # ---------------------------------------------------------------- capture mode: reply quality and slot outcome
    def window_quality(self, windows, results, counts, max_windows, params=None, quality=None, stream=None):
        """Quality records (rule: include/rfid_b200.h) of the stored windows of a `decode_capture` call: windows = the
        window tap it wrote (CUDA complex64 / float32 tensor of nseg * max_windows * len_epc samples), results / counts
        its outputs; params: `QualityParams` (None: defaults, see `default_quality_params`).  Asynchronous on `stream`.
        Returns quality, a CUDA uint8 tensor [nseg * max_windows, 16] (`quality_to_numpy` views it as QUALITY_DTYPE);
        slots beyond a segment's stored records are left as they were (zero when allocated here)."""
        import torch
        nseg = counts.numel()
        self._check_tap(windows, nseg, max_windows)
        if quality is None:
            quality = torch.zeros((nseg * max_windows, 16), dtype=torch.uint8, device=results.device)
        self._call("rfid_b200_window_quality", windows.data_ptr(), results.data_ptr(), counts.data_ptr(), nseg,
                   max_windows, _ref(params), quality.data_ptr(), _stream(stream, results.device))
        return quality

    def decode_capture_quality(self, iq, segs, max_windows=2, params=None, scale=SC16_SCALE):
        """`decode_capture` with the window tap set for this one call, then `window_quality` on what it wrote.  iq, segs
        and scale as in `decode_capture` (fc32 or sc16).  The tap takes nseg * max_windows * len_epc * 8 bytes of
        device memory (3.5 GB for 160,000 segments of 2 windows at 2 MS/s); it is released to torch's stream-ordered
        allocator on return, so the call stays asynchronous on the current stream like `decode_capture`.  Returns
        (results, counts, quality) as device tensors."""
        return self._decode_stages(iq, segs, max_windows, scale, params)[1][:3]

    def _decode_tapped(self, iq, segs, max_windows, scale):
        """`decode_capture` with a window tap set for this one call: (tap, results, counts)"""
        import torch
        nseg = segs.numel() * segs.element_size() // 16
        tap = torch.empty(nseg * max_windows * self.len_epc, dtype=torch.complex64, device=iq.device)
        self.set_window_tap(tap)
        try:
            results, counts = self.decode_capture(iq, segs, max_windows=max_windows, scale=scale)
        finally:
            self.set_window_tap(None)
        return tap, results, counts

    def _decode_stages(self, iq, segs, max_windows, scale, quality_params, recover=False, recover_params=None,
                       report=False, reject_empty=True, report_params=None, max_tags=1024):
        """`_decode_tapped`, then `window_quality`, `recover_epc` (recover) and `tag_report` (report) on what they
        wrote: (tap, (results, counts, quality, fixes, tags, summary, read_tag)), None for what a stage not run would
        give"""
        tap, results, counts = self._decode_tapped(iq, segs, max_windows, scale)
        quality = self.window_quality(tap, results, counts, max_windows, params=quality_params)
        fixes = self.recover_epc(tap, results, counts, quality, max_windows, params=recover_params) if recover else None
        tags = (None, None, None)
        if report:
            tags = self.tag_report(results, counts, segs, max_windows, quality=quality if reject_empty else None,
                                   fixes=fixes, params=report_params, max_tags=max_tags)
        return tap, (results, counts, quality, fixes) + tags

    # ---------------------------------------------------------------- capture mode: EPC replies that fail their CRC
    def recover_epc(self, windows, results, counts, quality, max_windows, params=None, fixes=None, stream=None):
        """Recovery records (rule: include/rfid_b200.h) of the stored windows of a `decode_capture` call: windows, results
        and counts as in `window_quality`, quality its output for them; params: `RecoverParams` (None: defaults, see
        `default_recover_params`).  Asynchronous on `stream`.  Returns fixes, a CUDA uint8 tensor [nseg * max_windows,
        32] (`fixes_to_numpy` views it as EPC_FIX_DTYPE); slots beyond a segment's stored records are left as they were
        (zero when allocated here).  `apply_fixes` folds the RECOVERED windows into the records."""
        import torch
        nseg = counts.numel()
        self._check_tap(windows, nseg, max_windows)
        if fixes is None:
            fixes = torch.zeros((nseg * max_windows, 32), dtype=torch.uint8, device=results.device)
        self._call("rfid_b200_recover_epc", windows.data_ptr(), results.data_ptr(), counts.data_ptr(),
                   quality.data_ptr(), nseg, max_windows, _ref(params), fixes.data_ptr(),
                   _stream(stream, results.device))
        return fixes

    def decode_capture_recover(self, iq, segs, max_windows=2, quality_params=None, recover_params=None,
                               scale=SC16_SCALE):
        """`decode_capture` with the window tap set for this one call, then `window_quality` and `recover_epc` on what it
        wrote; iq, segs and scale as in `decode_capture` (fc32 or sc16), the tap as in `decode_capture_quality`.
        Returns (results, counts, quality, fixes) as device tensors; the records are the decoder's, unchanged."""
        return self._decode_stages(iq, segs, max_windows, scale, quality_params, True, recover_params)[1][:4]

    # ---------------------------------------------------------------- capture mode: the tag inventory report
    def tag_report(self, results, counts, segs, max_windows, quality=None, fixes=None, params=None, max_tags=1024,
                   tags=None, summary=None, read_tag=None, stream=None):
        """The inventory report (rule: include/rfid_b200.h) of the stored slots of a `decode_capture` call: results,
        counts its outputs, segs the segment table it decoded (CUDA tensor, see `segments_to_device`); quality its
        `window_quality` records (None: no empty-slot rejection), fixes its `recover_epc` records (None: no recovered
        reads); params: `ReportParams` (None: defaults, see `default_report_params`).  Asynchronous on `stream`.  Returns
        (tags uint8[max_tags, 64], summary uint8[32], read_tag int32[nseg * max_windows]) as CUDA tensors, allocated here
        unless given (`tags_to_numpy` views the first two); read_tag entries of slots that are not stored are left as
        they were (-1 when allocated here)."""
        import torch
        nseg = counts.numel()
        if segs.numel() * segs.element_size() < nseg * 16:
            raise ValueError("the segment table holds fewer than nseg entries")
        dev = results.device
        if tags is None:
            tags = torch.zeros((max_tags, 64), dtype=torch.uint8, device=dev)
        if tags.numel() < max_tags * 64:
            raise ValueError("the tag buffer holds fewer than max_tags records")
        if summary is None:
            summary = torch.zeros(32, dtype=torch.uint8, device=dev)
        if read_tag is None:
            read_tag = torch.full((nseg * max_windows,), -1, dtype=torch.int32, device=dev)
        self._call("rfid_b200_tag_report", segs.data_ptr(), results.data_ptr(), counts.data_ptr(), nseg, max_windows,
                   _ptr(quality), _ptr(fixes), _ref(params), max_tags, tags.data_ptr() if max_tags > 0 else None,
                   summary.data_ptr(), read_tag.data_ptr(), _stream(stream, dev))
        return tags, summary, read_tag

    def decode_capture_report(self, iq, segs, max_windows=2, recover=True, reject_empty=True, quality_params=None,
                              recover_params=None, report_params=None, max_tags=1024, scale=SC16_SCALE):
        """`decode_capture` with the window tap set for this one call, then `window_quality`, `recover_epc` (recover=True)
        and `tag_report` on what they wrote; iq, segs and scale as in `decode_capture` (fc32 or sc16), the tap as in
        `decode_capture_quality`.  reject_empty: the report rejects reads in slots the quality rule calls EMPTY (CRC
        passes on noise; but also replies weaker than quality_params.empty_db, DESIGN 4.8).  Only the report has to
        come back to the host.  Returns (results, counts, quality, fixes, tags, summary, read_tag) as device tensors
        (fixes None without recovery)."""
        return self._decode_stages(iq, segs, max_windows, scale, quality_params, recover, recover_params, report=True,
                                   reject_empty=reject_empty, report_params=report_params, max_tags=max_tags)[1]

    # ---------------------------------------------------------------- capture mode: replies from tags you already know
    def match_epc(self, windows, results, counts, dictionary, max_windows, fixes=None, n_dict=None, params=None,
                  match=None, match_count=None, counts_per_entry=True, stream=None):
        """Attribution records (rule: include/rfid_b200.h) of the stored windows of a `decode_capture` call: windows,
        results and counts as in `window_quality`, fixes its `recover_epc` records (None: only CRC passes are already
        read); dictionary: uint8 [max_dict, 16] PC + EPC + CRC frames (a CUDA tensor, or host data copied to the device);
        n_dict: a CUDA int32 tensor whose first element is the live entry count (None: all max_dict); params:
        `MatchParams` (None: defaults, see `default_match_params`).  Asynchronous on `stream`.  Returns (match uint8
        [nseg * max_windows, 32], match_count uint8 [max_dict, 16] or None without counts_per_entry) as CUDA tensors;
        `matches_to_numpy` views them.  Match records of slots beyond a segment's stored records are left as they were
        (zero when allocated here)."""
        import torch
        nseg = counts.numel()
        dev = results.device
        self._check_tap(windows, nseg, max_windows)
        if not isinstance(dictionary, torch.Tensor):
            dictionary = torch.from_numpy(np.ascontiguousarray(dictionary, dtype=np.uint8).reshape(-1, 16)).to(dev)
        if dictionary.dtype != torch.uint8 or not dictionary.is_contiguous() or dictionary.numel() % 16:
            raise ValueError("the dictionary is a contiguous uint8 tensor of 16-byte frames")
        if dictionary.data_ptr() % 16:
            raise ValueError("the dictionary must be 16-byte aligned")
        max_dict = dictionary.numel() // 16
        if n_dict is not None and (n_dict.dtype != torch.int32 or n_dict.numel() < 1):
            raise ValueError("n_dict is a CUDA int32 tensor")
        if match is None:
            match = torch.zeros((nseg * max_windows, 32), dtype=torch.uint8, device=dev)
        if match_count is None and counts_per_entry:
            match_count = torch.empty((max_dict, 16), dtype=torch.uint8, device=dev)
        self._call("rfid_b200_match_epc", windows.data_ptr(), results.data_ptr(), counts.data_ptr(), _ptr(fixes), nseg,
                   max_windows, dictionary.data_ptr() if max_dict > 0 else None, _ptr(n_dict), max_dict, _ref(params),
                   match.data_ptr(), _ptr(match_count) if max_dict > 0 else None, _stream(stream, dev))
        return match, match_count

    def decode_capture_match(self, iq, segs, dictionary=None, max_windows=2, recover=True, reject_empty=True,
                             quality_params=None, recover_params=None, report_params=None, match_params=None,
                             max_tags=1024, scale=SC16_SCALE):
        """`decode_capture_report` (decode with the window tap, quality, recovery unless recover=False, the report), then
        `match_epc` on the same windows; iq, segs and scale as in `decode_capture` (fc32 or sc16).  dictionary None: the
        report's own tags -- their frames are copied on the device and the report's n_tags is the live count, so the
        call stays asynchronous.  Returns (results, counts, quality, fixes, tags, summary, read_tag, match, match_count)
        as device tensors (fixes None without recovery)."""
        import torch
        tap, out = self._decode_stages(iq, segs, max_windows, scale, quality_params, recover, recover_params,
                                       report=True, reject_empty=reject_empty, report_params=report_params,
                                       max_tags=max_tags)
        results, counts, _, fixes, tags, summary, _ = out
        n_dict = None
        if dictionary is None:
            dictionary = tags[:, :16].contiguous()
            n_dict = summary.view(torch.int32)[:1]
        return out + self.match_epc(tap, results, counts, dictionary, max_windows, fixes=fixes, n_dict=n_dict,
                                    params=match_params)

    # ---------------------------------------------------------------- capture ingest
    def segment_capture(self, iq, segmenter=None, capacity=None, stream=None, scale=SC16_SCALE):
        """CW-gap segment table (SEGMENT_DTYPE ndarray) of a CUDA capture tensor (complex64 / float32 interleaved, or an
        sc16 torch.int16 tensor as in `decode_capture`, whose table is that of its conversion)."""
        fmt, cap_args = _capture(iq, scale)
        cap = int(capacity) if capacity is not None else max(16, cap_args[1] // 4096)
        segs = np.zeros(cap, dtype=abi.SEGMENT_DTYPE)
        n = C.c_int(0)
        self._call("rfid_b200_segment_capture" + fmt, *cap_args, _ref(segmenter), segs.ctypes.data, cap, C.byref(n),
                   _stream(stream, iq.device))
        return segs[:n.value].copy()

    def ingest_capture_host(self, iq, segmenter=None, max_windows=4, capacity=None, scale=SC16_SCALE):
        """Recorded capture -> (segs, records, counts).  iq: host complex64 ndarray (e.g. np.fromfile / np.memmap of an
        fc32 file), or an np.int16 array of interleaved I, Q (an sc16 file, e.g. np.memmap(path, dtype=np.int16)),
        decoded as its conversion I * scale, Q * scale."""
        sc16 = np.asarray(iq).dtype == np.int16
        raw = np.ascontiguousarray(iq).ravel() if sc16 else np.ascontiguousarray(iq).view(np.float32).ravel()
        if raw.size % 2:
            raise ValueError("an interleaved I, Q capture has an even number of values")
        n_raw = raw.size // 2
        cap = int(capacity) if capacity is not None else max(16, n_raw // 4096)
        segs = np.zeros(cap, dtype=abi.SEGMENT_DTYPE)
        recs = np.zeros((cap, max_windows), dtype=abi.RESULT_DTYPE)
        counts = np.zeros(cap, dtype=np.int32)
        n = C.c_int(0)
        head = (n_raw, scale) if sc16 else (n_raw,)
        self._call("rfid_b200_ingest_capture_host" + ("_sc16" if sc16 else ""), raw.ctypes.data, *head, _ref(segmenter),
                   max_windows, segs.ctypes.data, cap, C.byref(n), recs.ctypes.data, counts.ctypes.data)
        k = n.value
        return segs[:k].copy(), recs[:k].copy(), counts[:k].copy()

    # ---------------------------------------------------------------- TX synthesiser / slot simulator
    def tx_synth(self, script, dac_rate=1000000, device="cuda:0"):
        """script: iterable of (kind, arg) -> float32 CUDA tensor with the reader's TX envelope."""
        import torch
        scr = np.array([(int(k), int(a)) for k, a in script], dtype=abi.TX_COMMAND_DTYPE)
        n = C.c_size_t(0)
        self._call("rfid_b200_tx_synth", scr.ctypes.data, scr.size, dac_rate, None, 0, C.byref(n), None)
        out = torch.empty(n.value, dtype=torch.float32, device=device)
        self._call("rfid_b200_tx_synth", scr.ctypes.data, scr.size, dac_rate, out.data_ptr(), out.numel(), C.byref(n),
                   _stream(None, out.device))
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
        self._call("rfid_b200_sim_capture", C.byref(sim), first_segment, nseg, iq.data_ptr(), segs.data_ptr(),
                   truth.data_ptr(), _stream(None, dev))
        return {"iq": iq, "segs": segs, "truth": truth, "segment_len": seg_len}

    def set_window_tap(self, tensor_or_none):
        self._call("rfid_b200_set_window_tap", _ptr(tensor_or_none))

    def enable_kernel_timing(self, on=True):
        self._call("rfid_b200_enable_kernel_timing", int(on))

    def kernel_time(self, reset=True):
        ms, n = C.c_float(0), C.c_int(0)
        self._call("rfid_b200_kernel_time", int(reset), C.byref(ms), C.byref(n))
        return ms.value, n.value

    def last_launch_count(self):
        return self.lib.rfid_b200_last_launch_count(self.h)

    def reduce_stats(self, recs, counts, continuous):
        recs = np.ascontiguousarray(recs, dtype=abi.RESULT_DTYPE)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        nseg = counts.size
        max_per = recs.size // nseg if nseg else 1
        st = abi.Stats()
        self._call("rfid_b200_reduce_stats", recs.ctypes.data, counts.ctypes.data, nseg, max(1, max_per),
                   int(bool(continuous)), C.byref(st))
        return st

    # ---------------------------------------------------------------- block mode
    def gate_work(self, chunk, seek=0, want_magn2=False):
        x = np.ascontiguousarray(chunk, dtype=np.complex64)
        n = x.size
        out = np.zeros(max(n, 1), dtype=np.complex64)
        m2 = np.zeros(max(n, 1), dtype=np.float32) if want_magn2 else None
        c, w, cl = C.c_int(0), C.c_int(0), C.c_int(0)
        self._call("rfid_b200_gate_work", int(seek), x.ctypes.data, n, out.ctypes.data, max(n, 1), C.byref(c),
                   C.byref(w), C.byref(cl), m2.ctypes.data if want_magn2 else None)
        res = {"consumed": c.value, "written": w.value, "closed": cl.value, "out": out[:w.value]}
        if want_magn2:
            res["magn2"] = m2[:w.value]
        return res

    def decoder_work(self, kind, window):
        w = np.ascontiguousarray(window, dtype=np.complex64)
        rec = np.zeros(1, dtype=abi.RESULT_DTYPE)
        bits = np.zeros(128, dtype=np.float32)
        self._call("rfid_b200_decoder_work", int(kind), w.ctypes.data, w.size, rec.ctypes.data, bits.ctypes.data)
        return rec[0], bits[:16 if kind == abi.RN16 else 128]

    def mf_work(self, chunk):
        x = np.ascontiguousarray(chunk, dtype=np.complex64)
        cap = x.size // self.params.decim + 2
        out = np.zeros(cap, dtype=np.complex64)
        w = C.c_int(0)
        self._call("rfid_b200_mf_work", x.ctypes.data, x.size, out.ctypes.data, cap, C.byref(w))
        return out[:w.value]


def segments_to_device(segs, device):
    """SEGMENT_DTYPE ndarray -> CUDA uint8 tensor holding the same bytes."""
    import torch
    b = np.ascontiguousarray(segs, dtype=abi.SEGMENT_DTYPE).view(np.uint8)
    return torch.from_numpy(b.copy()).to(device)


def _records_to_numpy(records, counts, per_segment, dtype):
    """device uint8[nseg*per_segment,dtype.itemsize] + int32[nseg] -> (dtype[nseg,per_segment], int32[nseg])"""
    r = records.cpu().numpy().reshape(-1).view(dtype)
    c = counts.cpu().numpy()
    return r.reshape(c.size, per_segment), c


def results_to_numpy(results, counts, max_windows):
    """device uint8[nseg*max_windows,64] + int32[nseg] -> (RESULT_DTYPE[nseg,max_windows], int32[nseg])"""
    return _records_to_numpy(results, counts, max_windows, abi.RESULT_DTYPE)


def commands_to_numpy(cmds, counts, max_commands):
    """device uint8[nseg*max_commands,64] + int32[nseg] -> (COMMAND_DTYPE[nseg,max_commands], int32[nseg])"""
    return _records_to_numpy(cmds, counts, max_commands, abi.COMMAND_DTYPE)


#: one row per stored tag window: the reader command that armed it (see `transcript`)
TRANSCRIPT_DTYPE = np.dtype([("segment", "<i4"), ("window", "<i4"), ("kind", "<i4"), ("command", "<i4"),
                             ("cmd_kind", "<i4"), ("cmd_arg", "<i4"), ("ack_echo", "<i4"), ("turnaround_us", "<f8")])


def transcript(cmds, cmd_counts, recs, counts, decim=5, adc_rate=2_000_000):
    """Pair every stored tag window with the reader command that armed it (host numpy only).

    cmds, cmd_counts: `decode_commands` output (COMMAND_DTYPE[nseg, max_commands]); recs, counts: `decode_capture` output
    (RESULT_DTYPE[nseg, max_windows]) of the same segment table.  Per window:
      command        index of the last stored command of the segment with end <= open_index*decim (raw samples), or -1;
      cmd_kind/arg   that command's kind and arg (-1 without one);
      ack_echo       EPC windows: 1 if the arming command is an ACK whose arg equals the tag_id of the segment's preceding
                     RN16 window, else 0; RN16 windows: -1;
      turnaround_us  EPC windows armed by an ACK that follows an RN16 window: from the RN16 window's end,
                     (open_index + length)*decim, to the ACK's start, in microseconds at adc_rate; NaN otherwise.
    """
    cmds = np.asarray(cmds, dtype=abi.COMMAND_DTYPE)
    recs = np.asarray(recs, dtype=abi.RESULT_DTYPE)
    cmd_counts = np.asarray(cmd_counts)
    counts = np.asarray(counts)
    rows = []
    for s in range(counts.size):
        cs = cmds[s, :max(0, min(int(cmd_counts[s]), cmds.shape[1]))]
        ends = cs["end"].astype(np.int64)
        prev_rn16 = None
        for w in recs[s, :max(0, min(int(counts[s]), recs.shape[1]))]:
            r = np.zeros((), dtype=TRANSCRIPT_DTYPE)
            r["segment"], r["window"], r["kind"] = s, w["window"], w["kind"]
            k = int(np.searchsorted(ends, int(w["open_index"]) * decim, side="right")) - 1 if cs.size else -1
            # (ends are increasing: commands do not overlap)
            r["command"] = k
            r["cmd_kind"] = cs["kind"][k] if k >= 0 else -1
            r["cmd_arg"] = cs["arg"][k] if k >= 0 else -1
            r["ack_echo"] = -1
            r["turnaround_us"] = np.nan
            if int(w["kind"]) == abi.EPC:
                is_ack = k >= 0 and int(cs["kind"][k]) == abi.TX_ACK
                r["ack_echo"] = int(is_ack and prev_rn16 is not None and int(cs["arg"][k]) == int(prev_rn16["tag_id"]))
                if is_ack and prev_rn16 is not None:
                    rn16_end = (int(prev_rn16["open_index"]) + int(prev_rn16["length"])) * decim
                    r["turnaround_us"] = (int(cs["start"][k]) - rn16_end) * 1e6 / adc_rate
            else:
                prev_rn16 = w
            rows.append(r)
    return np.array(rows, dtype=TRANSCRIPT_DTYPE)


def quality_to_numpy(quality, counts, max_windows):
    """device uint8[nseg*max_windows,16] + int32[nseg] -> (QUALITY_DTYPE[nseg,max_windows], int32[nseg])"""
    return _records_to_numpy(quality, counts, max_windows, abi.QUALITY_DTYPE)


def fixes_to_numpy(fixes, counts, max_windows):
    """device uint8[nseg*max_windows,32] + int32[nseg] -> (EPC_FIX_DTYPE[nseg,max_windows], int32[nseg])"""
    return _records_to_numpy(fixes, counts, max_windows, abi.EPC_FIX_DTYPE)


def apply_fixes(recs, counts, fixes):
    """A copy of the records (RESULT_DTYPE[nseg, max_windows], host numpy) in which every stored RECOVERED window
    (`recover_epc` output, EPC_FIX_DTYPE[nseg, max_windows]) has the corrected bits, crc_ok = 1 and tag_id = bits
    104..111, as the decoder sets them for a passing EPC; `reduce_stats`, `transcript` and `slot_table` then count
    recovered reads like any other."""
    out = np.array(recs, dtype=abi.RESULT_DTYPE, copy=True)
    fixes = np.asarray(fixes, dtype=abi.EPC_FIX_DTYPE)
    counts = np.asarray(counts)
    stored = np.arange(out.shape[1])[None, :] < np.minimum(np.maximum(counts, 0), out.shape[1])[:, None]
    fix = stored & (fixes["status"] == abi.FIX_RECOVERED)
    out["bits"][fix] = fixes["bits"][fix]
    out["crc_ok"][fix] = 1
    out["tag_id"][fix] = fixes["bits"][fix][:, 13]
    return out


def tags_to_numpy(tags, summary):
    """`tag_report` output -> (TAG_DTYPE[min(n_tags, max_tags)], TAG_SUMMARY_DTYPE record)"""
    sm = summary.cpu().numpy().reshape(-1).view(abi.TAG_SUMMARY_DTYPE)[0]
    t = tags.cpu().numpy().reshape(-1).view(abi.TAG_DTYPE)
    return t[:min(int(sm["n_tags"]), t.size)].copy(), sm


#: one row per tag of a report, in display units (see `tag_table`)
TAG_TABLE_DTYPE = np.dtype([("epc", "U32"), ("reads", "<i4"), ("recovered", "<i4"), ("first_us", "<f8"),
                            ("last_us", "<f8"), ("peak_rssi_db", "<f8"), ("last_phase_deg", "<f8")])


def matches_to_numpy(match, counts, max_windows, match_count=None):
    """`match_epc` output -> (EPC_MATCH_DTYPE[nseg, max_windows], MATCH_COUNT_DTYPE[max_dict] or None)"""
    m = _records_to_numpy(match, counts, max_windows, abi.EPC_MATCH_DTYPE)[0]
    mc = match_count.cpu().numpy().reshape(-1).view(abi.MATCH_COUNT_DTYPE) if match_count is not None else None
    return m, mc


def tag_table(tags, ntaps=25, adc_rate=2_000_000, matched=None):
    """The report's tags (TAG_DTYPE rows) in display units (host numpy only): PC + EPC + CRC as hex, reads, recovered,
    first and last seen in microseconds from the capture's first sample (the times are raw samples at adc_rate),
    peak_rssi_db = 10 log10(peak_power / ntaps^2), the strongest reply's power in dB relative to a full-scale sample (h
    is a sum over the matched filter's ntaps samples), and last_phase_deg = arg(last h) in degrees.  matched: per tag,
    the failing replies `match_epc` attributed to it (e.g. `match_count["matched"]` of a match against the report's
    own tags); given, the table gains a `matched` column after `recovered`."""
    tags = np.asarray(tags, dtype=abi.TAG_DTYPE)
    if matched is not None:
        matched = np.asarray(matched).reshape(-1)
        if matched.size < tags.size:
            raise ValueError("matched holds fewer entries than there are tags")
        names = TAG_TABLE_DTYPE.names
        i = names.index("recovered") + 1
        dt = np.dtype([(n, TAG_TABLE_DTYPE[n]) for n in names[:i]] + [("matched", "<i4")] +
                      [(n, TAG_TABLE_DTYPE[n]) for n in names[i:]])
        out = np.zeros(tags.size, dtype=dt)
        out["matched"] = matched[:tags.size]
    else:
        out = np.zeros(tags.size, dtype=TAG_TABLE_DTYPE)
    out["epc"] = [bytes(bytearray(e)).hex() for e in tags["epc"]]
    out["reads"], out["recovered"] = tags["reads"], tags["recovered"]
    out["first_us"] = tags["first_time"] * 1e6 / adc_rate
    out["last_us"] = tags["last_time"] * 1e6 / adc_rate
    with np.errstate(divide="ignore", invalid="ignore"):
        out["peak_rssi_db"] = 10.0 * np.log10(tags["peak_power"].astype(np.float64) / float(ntaps) ** 2)
    out["last_phase_deg"] = np.degrees(np.arctan2(tags["last_h_im"].astype(np.float64),
                                                  tags["last_h_re"].astype(np.float64)))
    return out


#: one row per segment: what its RN16 and EPC windows say about the slot (see `slot_table`)
SLOT_DTYPE = np.dtype([("segment", "<i4"), ("rn16_outcome", "<i4"), ("epc_outcome", "<i4"), ("tag_id", "<i4"),
                       ("crc_ok", "<i4"), ("rn16_energy_db", "<f8"), ("rn16_snr_db", "<f8"), ("epc_energy_db", "<f8"),
                       ("epc_snr_db", "<f8")])


def _db(x):
    with np.errstate(divide="ignore", invalid="ignore"):
        return 10.0 * np.log10(np.float64(x))


def slot_table(recs, counts, quality):
    """One row per segment of a capture decoded one slot per segment (host numpy only).  recs, counts: `decode_capture`
    output (RESULT_DTYPE[nseg, max_windows]); quality: `window_quality` output (QUALITY_DTYPE[nseg, max_windows]).  The
    slot's RN16 window is the segment's first stored window, its EPC window the second.  Outcomes are RFID_B200_SLOT_*
    or -1 where the segment has no such window; tag_id and crc_ok come from the EPC record (-1 without one); energy and
    SNR in dB (NaN without a window)."""
    recs = np.asarray(recs, dtype=abi.RESULT_DTYPE)
    quality = np.asarray(quality, dtype=abi.QUALITY_DTYPE)
    counts = np.asarray(counts)
    out = np.zeros(counts.size, dtype=SLOT_DTYPE)
    out["segment"] = np.arange(counts.size)
    for f in ("rn16_outcome", "epc_outcome", "tag_id", "crc_ok"):
        out[f] = -1
    for f in ("rn16_energy_db", "rn16_snr_db", "epc_energy_db", "epc_snr_db"):
        out[f] = np.nan
    n = np.minimum(np.maximum(counts, 0), recs.shape[1])
    for k, name in ((0, "rn16"), (1, "epc")):
        has = n > k
        if k >= recs.shape[1] or not has.any():
            continue
        q = quality[has, k]
        out[name + "_outcome"][has] = q["outcome"]
        out[name + "_energy_db"][has] = _db(q["energy"])
        out[name + "_snr_db"][has] = _db(q["snr"])
        if name == "epc":
            out["tag_id"][has] = recs[has, k]["tag_id"]
            out["crc_ok"][has] = recs[has, k]["crc_ok"]
    return out


def inventory_summary(recs, counts, quality):
    """Counts of an inventory's slots from `slot_table`: empty, single and collided slots (RN16 outcome; segments
    without an RN16 window are not counted), and the single slots whose EPC passed its CRC."""
    t = slot_table(recs, counts, quality)
    rn = t["rn16_outcome"]
    return {"slots": int((rn >= 0).sum()), "empty": int((rn == abi.SLOT_EMPTY).sum()),
            "single": int((rn == abi.SLOT_SINGLE).sum()), "collision": int((rn == abi.SLOT_COLLISION).sum()),
            "single_epc_ok": int(((rn == abi.SLOT_SINGLE) & (t["crc_ok"] == 1)).sum())}
