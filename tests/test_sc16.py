"""Complex int16 (sc16) captures: decoded in the capture kernels' load stage, bit-identical to decoding their float
conversion ((float)I * scale, (float)Q * scale) through the fc32 path, and through it to the restatement and the
reference's own blocks.

The sc16 fixture is the reference's recording quantised to int16 (scales 1/32767 and 2^-15); the CPU test below checks
that the quantisation leaves every decision of the recording as it was.
"""
import ctypes as C
import sys

import numpy as np
import pytest

from conftest import GOLDEN, records_equal
from gen2_uhf_rfid_reader_b200 import abi, synth

sys.path.insert(0, GOLDEN)
from make_golden import rate_capture  # noqa: E402

SCALES = (float(np.float32(1.0 / 32767.0)), 2.0 ** -15)
INT_FIELDS = ("open_index", "length", "kind", "sync_index", "crc_ok", "tag_id", "bits", "T")


def quantise(iq, scale):
    """complex64 ndarray -> interleaved int16 I, Q: round(x / scale), clamped"""
    x = np.ascontiguousarray(iq).view(np.float32).ravel()
    return np.clip(np.rint(x / np.float32(scale)), -32768, 32767).astype(np.int16)


def convert(q, scale):
    """the fc32 capture an sc16 capture stands for: np.float32(i) * np.float32(scale), one rounding per component"""
    return (q.astype(np.float32) * np.float32(scale)).view(np.complex64)


def _assert_same(got, ref, what=""):
    bad = records_equal(got, ref)
    assert not bad, "%s fields differ: %s" % (what, bad)


# ------------------------------------------------------------------ CPU: the fixture
@pytest.mark.parametrize("scale", SCALES, ids=["1_32767", "2^-15"])
def test_quantised_recording_decodes_like_the_float_recording(oracle, cfg1_iq, cfg1_golden, scale):
    """the recording quantised to int16 and converted back decodes, in the restatement, to the same decisions and
    READER_STATS as the reference run on the float recording (scores move: the input changed)"""
    q = quantise(cfg1_iq, scale)
    x = convert(q, scale)
    assert x.size == cfg1_iq.size and not np.array_equal(x, cfg1_iq)
    recs, n = oracle.decode_stream(x)
    assert n == 142
    for f in INT_FIELDS:
        assert recs[f].tobytes() == cfg1_golden[f].tobytes(), f
    rel = np.abs(recs["score"] - cfg1_golden["score"]) / cfg1_golden["score"]
    assert 0 < rel.max() < 1e-3
    st = oracle.reduce_stats(recs[None, :], np.array([n], dtype=np.int32), continuous=True)
    ref = oracle.reduce_stats(cfg1_golden[None, :], np.array([142], dtype=np.int32), continuous=True)
    assert bytes(st) == bytes(ref)
    assert st.n_epc_correct == 70


# ------------------------------------------------------------------ GPU
def _rx(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx(**kw)


@pytest.fixture(scope="module")
def rx():
    return _rx()


def _decode_sc16(rx, q, segs, scale, max_windows):
    """device-resident sc16 decode of host int16 q with a host segment table -> (records, counts)"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    dev = torch.device("cuda:0")
    iq = torch.from_numpy(q.copy()).to(dev)
    dsegs = capi.segments_to_device(segs, dev)
    res, cnt = rx.decode_capture(iq, dsegs, max_windows=max_windows, scale=scale)
    torch.cuda.synchronize()
    return capi.results_to_numpy(res, cnt, max_windows)


def _check_sc16(rx, oracle, q, segs, scale, max_windows, what, oracle_check=True):
    """sc16 records = fc32 records of the conversion = the restatement's records of the conversion"""
    recs, counts = _decode_sc16(rx, q, segs, scale, max_windows)
    x = convert(q, scale)
    frecs, fcounts = rx.decode_capture_host(x, segs, max_windows=max_windows)
    assert counts.tolist() == fcounts.tolist(), what
    _assert_same(recs, frecs, what + ": sc16 vs fc32")
    if oracle_check:
        orecs, ocounts, _ = oracle.decode_segments(x, segs, max_per_seg=max_windows)
        assert counts.tolist() == ocounts.tolist(), what
        _assert_same(recs, orecs, what + ": sc16 vs restatement")
    return recs, counts


@pytest.mark.gpu
def test_device_conversion_is_exact_for_every_int16():
    """RawSc16::cvt (the kernels' conversion) = np.float32(i) * np.float32(scale) for all 65,536 int16 values in both
    half-words; scale 1 checks the int16 -> float step alone"""
    import torch
    from gen2_uhf_rfid_reader_b200.build import SC16_HARNESS, SC16_HARNESS_SRC, build_harness
    h = C.CDLL(build_harness(SC16_HARNESS_SRC, SC16_HARNESS))
    h.sc16_harness_convert.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    scales = np.array(SCALES + (1.0, 3.0517578125e-05 * 3, 1e-3), dtype=np.float32)
    d_scales = torch.from_numpy(scales).cuda()
    out = torch.empty((scales.size, 65536, 2), dtype=torch.float32, device="cuda")
    assert h.sc16_harness_convert(d_scales.data_ptr(), scales.size, out.data_ptr()) == 0
    got = out.cpu().numpy()
    i = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    qv = ~i
    for k, s in enumerate(scales):
        want_i = i.astype(np.float32) * s
        want_q = qv.astype(np.float32) * s
        assert got[k, :, 0].tobytes() == want_i.tobytes(), s
        assert got[k, :, 1].tobytes() == want_q.tobytes(), s


@pytest.mark.gpu
@pytest.mark.parametrize("scale", SCALES, ids=["1_32767", "2^-15"])
def test_recording_continuous_and_sliced(rx, oracle, cfg1_iq, scale):
    """the sc16 recording as one segment (against the reference's blocks too), and cut into slices whose offsets take
    every residue mod 8, with ragged ends and a last slice that ends on the capture's last sample (1,247,958 samples:
    2 mod 4, so the loader's plain-load tail runs)"""
    from oracle.refflow import RefFlow
    q = quantise(cfg1_iq, scale)
    n = cfg1_iq.size
    recs, counts = _check_sc16(rx, oracle, q, abi.make_segments([0], [n]), scale, 256, "whole")
    assert counts[0] == 142
    ref = RefFlow(0).run_stream(convert(q, scale))
    assert ref["n_windows"] == 142
    _assert_same(recs[0, :142], ref["records"], "whole: sc16 vs reference blocks")
    rng = np.random.default_rng(int(scale * 1e9) % 1000)
    offs = [int(o) for o in rng.integers(0, n - 60000, size=40)]
    offs = [o - o % 8 + r for o, r in zip(offs, list(range(8)) * 5)]
    lens = [int(v) for v in rng.integers(20000, 60000, size=40)]
    offs += [n - 70001, n - 3, n - 1]
    lens += [70001, 3, 1]
    _check_sc16(rx, oracle, q, abi.make_segments(offs, lens), scale, 16, "slices")


def _kernel_names(fn):
    """names of the capture kernels fn() launched (torch.profiler, CUDA activity only)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = set()
    for e in prof.events():
        for k in ("rx_pack_kernel", "rx_fused_split_kernel", "rx_fused_kernel"):
            if k in e.name:
                names.add(k)
    return names


def _ragged(segs, seed):
    """every offset residue mod 8 and ragged lengths on a capture's own segment table, plus empty and tiny segments"""
    rng = np.random.default_rng(seed)
    s = segs.copy()
    s["offset"] = s["offset"] + (np.arange(s.size) % 8).astype(np.uint64)
    s["length"] = (s["length"] - rng.integers(8, 3000, size=s.size)).astype(np.uint32)
    extra = abi.make_segments([int(s["offset"][0]) + k for k in range(5)], [0, 1, 3, 7, 600])
    return np.concatenate([s, extra])


KERNEL_CASES = [
    # (id, adc, ntaps, RFID_B200_PACK_G, RFID_B200_KERNEL, expected kernel)
    ("pack-2.0-G1", 2_000_000, 25, "1", None, "rx_pack_kernel"),
    ("pack-2.0-G3", 2_000_000, 25, "3", None, "rx_pack_kernel"),
    ("pack-2.0-G8", 2_000_000, 25, "8", None, "rx_pack_kernel"),
    ("pack-1.2-G1", 1_200_000, 25, "1", None, "rx_pack_kernel"),
    ("pack-1.2-G3", 1_200_000, 25, "3", None, "rx_pack_kernel"),
    ("pack-1.2-G8", 1_200_000, 25, "8", None, "rx_pack_kernel"),
    ("split-2.0-forced", 2_000_000, 25, None, "split", "rx_fused_split_kernel"),
    ("split-0.4", 400_000, 25, None, None, "rx_fused_split_kernel"),
    ("split-1.0", 1_000_000, 25, None, None, "rx_fused_split_kernel"),
    ("split-1.0-12taps", 1_000_000, 12, None, None, "rx_fused_split_kernel"),
    ("fused-2.6", 2_600_000, 25, None, None, "rx_fused_kernel"),
    ("fused-4.0", 4_000_000, 50, None, None, "rx_fused_kernel"),
    ("fused-8.0", 8_000_000, 100, None, None, "rx_fused_kernel"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_every_kernel_in_sc16(oracle, case, monkeypatch):
    """each capture kernel on quantised captures (segment offsets of every residue mod 8, ragged ends, empty and tiny
    segments): the same kernel as fc32, records = fc32 on the conversion = the restatement"""
    import torch
    from oracle.pyoracle import Oracle
    from gen2_uhf_rfid_reader_b200 import capi
    key, adc, ntaps, g, kern, want = case
    if g:
        monkeypatch.setenv("RFID_B200_PACK_G", g)
    if kern:
        monkeypatch.setenv("RFID_B200_KERNEL", kern)
    rxk = _rx(adc_rate=adc, ntaps=ntaps)
    cap = synth.make_capture(24, seed=31, adc_rate=adc) if adc == 2_000_000 else rate_capture(adc, {})
    scale = SCALES[0]
    q = quantise(cap["iq"].numpy(), scale)
    segs = _ragged(cap["segments"], adc // 1000 + ntaps)
    dev = torch.device("cuda:0")
    iq = torch.from_numpy(q.copy()).to(dev)
    dsegs = capi.segments_to_device(segs, dev)
    assert _kernel_names(lambda: rxk.decode_capture(iq, dsegs, max_windows=4, scale=scale)) == {want}
    assert _kernel_names(lambda: rxk.decode_capture_host(convert(q, scale), segs, max_windows=4)) == {want}
    o = oracle if (adc, ntaps) == (2_000_000, 25) else Oracle(adc_rate=adc, ntaps=ntaps)
    _, counts = _check_sc16(rxk, o, q, segs, scale, 4, key)
    assert counts.sum() >= 10
    # a capture whose length is not a multiple of 4 samples, with a segment that ends on its last sample
    for cut in (1, 2, 3):
        n = q.size // 2 - cut
        n -= n % 4 == 0
        qn = q[:2 * n]
        tail = abi.make_segments([int(cap["segments"]["offset"][-1]) + cut, n - 7, n - 1],
                                 [n - int(cap["segments"]["offset"][-1]) - cut, 7, 1])
        _check_sc16(rxk, o, qn, tail, scale, 4, "%s tail %d" % (key, cut))


@pytest.mark.gpu
def test_cfg2_full_size_sc16_equals_fc32_and_truth(rx):
    """1000 simulated slots quantised on the GPU: sc16 = fc32 of the conversion bit for bit, decisions = truth"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    sim = capi.default_sim()
    cap = rx.sim_capture(sim, 1000)
    scale = SCALES[0]
    q = torch.round(torch.view_as_real(cap["iq"]) / scale).clamp(-32768, 32767).to(torch.int16)
    x = torch.view_as_complex((q.float() * scale).contiguous())
    res, cnt = rx.decode_capture(q, cap["segs"], max_windows=2, scale=scale)
    fres, fcnt = rx.decode_capture(x, cap["segs"], max_windows=2)
    torch.cuda.synchronize()
    recs, counts = capi.results_to_numpy(res, cnt, 2)
    frecs, fcounts = capi.results_to_numpy(fres, fcnt, 2)
    assert counts.tolist() == fcounts.tolist()
    _assert_same(recs, frecs, "cfg2 sc16 vs fc32")
    truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
    assert (counts == 2).all()
    assert (recs[:, 0]["tag_id"] == truth["strongest_rn16"]).all()
    assert (recs[:, 1]["crc_ok"] == 1).all() and (recs[:, 1]["bits"] == truth["epc"]).all()


def _flatten(recs, counts, segs, decim=5):
    out = []
    for s in range(len(counts)):
        r = recs[s, :counts[s]].copy()
        r["open_index"] += int(segs[s]["offset"]) // decim
        out.append(r)
    return np.concatenate(out)


@pytest.mark.gpu
def test_ingest_sc16_recording(rx, cfg1_iq, cfg1_golden):
    """ingest of the int16 recording (pageable and pinned) and segment_capture of it on the device: the segment table
    of the fc32 conversion and of the segmenter model, the same records, and the continuous reference run's decisions"""
    import torch
    import segmenter_model as sm
    scale = SCALES[0]
    q = quantise(cfg1_iq, scale)
    x = convert(q, scale)
    want, _ = sm.segment_table(x)
    fsegs, frecs, fcounts = rx.ingest_capture_host(x, max_windows=4)
    assert [(int(s["offset"]), int(s["length"])) for s in fsegs] == want and len(want) == 72
    pinned = torch.empty(q.size, dtype=torch.int16, pin_memory=True)
    pinned.numpy()[:] = q
    for src in (q, pinned.numpy()):
        segs, recs, counts = rx.ingest_capture_host(src, max_windows=4, scale=scale)
        assert segs.tobytes() == fsegs.tobytes()
        assert counts.tolist() == fcounts.tolist()
        _assert_same(recs, frecs, "ingest sc16 vs fc32")
    flat = _flatten(recs, counts, segs)
    assert len(flat) == 142
    for f in INT_FIELDS:
        assert flat[f].tobytes() == cfg1_golden[f].tobytes(), f
    dsegs = rx.segment_capture(torch.from_numpy(q.reshape(-1, 2).copy()).cuda(), scale=scale)
    assert dsegs.tobytes() == fsegs.tobytes()


@pytest.mark.gpu
def test_sc16_argument_checks(rx):
    """scale 0, negative, NaN, inf and a device pointer that is not 16-byte aligned: RFID_B200_EINVAL, and the wrapper
    raises"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    q = torch.zeros(2 * 4096 + 8, dtype=torch.int16, device="cuda")
    segs = capi.segments_to_device(abi.make_segments([0], [4000]), "cuda")
    res = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    hs = np.zeros(16, dtype=abi.SEGMENT_DTYPE)
    n = C.c_int(0)
    hq = np.zeros(2 * 4096, dtype=np.int16)
    hr = np.zeros((16, 4), dtype=abi.RESULT_DTYPE)
    hc = np.zeros(16, dtype=np.int32)
    for bad in (0.0, -1.0 / 32767, float("nan"), float("inf"), float("-inf")):
        assert L.rfid_b200_decode_capture_sc16(rx.h, q.data_ptr(), 4096, bad, segs.data_ptr(), 1, 4, res.data_ptr(),
                                               cnt.data_ptr(), None) == abi.EINVAL
        assert L.rfid_b200_segment_capture_sc16(rx.h, q.data_ptr(), 4096, bad, None, hs.ctypes.data, 16, C.byref(n),
                                                None) == abi.EINVAL
        assert L.rfid_b200_ingest_capture_host_sc16(rx.h, hq.ctypes.data, 4096, bad, None, 4, hs.ctypes.data, 16,
                                                    C.byref(n), hr.ctypes.data, hc.ctypes.data) == abi.EINVAL
        with pytest.raises(capi.RfidB200Error):
            rx.decode_capture(q, segs, max_windows=4, scale=bad)
        with pytest.raises(capi.RfidB200Error):
            rx.segment_capture(q, scale=bad)
        with pytest.raises(capi.RfidB200Error):
            rx.ingest_capture_host(hq, scale=bad)
    for shift in (2, 4, 6):   # 4, 8 and 12 bytes off a 16-byte boundary
        mis = q[shift:shift + 2 * 4096]
        assert mis.data_ptr() % 16 != 0
        assert L.rfid_b200_decode_capture_sc16(rx.h, mis.data_ptr(), 4096, SCALES[0], segs.data_ptr(), 1, 4,
                                               res.data_ptr(), cnt.data_ptr(), None) == abi.EINVAL
        assert L.rfid_b200_segment_capture_sc16(rx.h, mis.data_ptr(), 4096, SCALES[0], None, hs.ctypes.data, 16,
                                                C.byref(n), None) == abi.EINVAL
        with pytest.raises(capi.RfidB200Error):
            rx.decode_capture(mis, segs, max_windows=4)
    with pytest.raises(ValueError):
        rx.decode_capture(q.reshape(-1, 4), segs, max_windows=4)
    torch.cuda.synchronize()
