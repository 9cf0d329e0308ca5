"""GPU tests at sample rates other than 2 MS/s (run with -m gpu on an H100).

Every kernel the library picks is compared, bit for bit, with the reference's own blocks (stored outputs in
tests/golden/reference_rates.npz) and with the C restatement, at one or more rates per kernel: rx_fused_split_kernel<5,0>
and <5,5> at 1.0 MS/s, rx_pack_kernel at 1.2 MS/s (25 taps), rx_fused_split_kernel<5,5> at 1.4 - 2.4 MS/s, rx_fused_kernel
from 2.6 MS/s up.  At 1.2 MS/s the packed kernel runs code the 2 MS/s configuration never reaches: n_T1 + 1 < 64 in the
closed-run scan, a DC divisor (28) without the verified fast division, and a DC lookback of 7 lanes instead of 12.
"""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, records_equal
from gen2_uhf_rfid_reader_b200 import abi, synth

sys.path.insert(0, GOLDEN)
from make_golden import RATE_VARIANTS, RATES, rate_capture, rate_cases  # noqa: E402

pytestmark = pytest.mark.gpu

R12 = 1_200_000   # the packed kernel's second rate


@pytest.fixture(scope="module")
def ref_rates():
    with np.load(os.path.join(GOLDEN, "reference_rates.npz")) as z:
        return {k: z[k] for k in z.files}


_RX, _OR = {}, {}


def rx_for(adc, ntaps=25, fixed_q=0):
    from gen2_uhf_rfid_reader_b200 import capi
    key = (adc, ntaps, fixed_q)
    if key not in _RX:
        _RX[key] = capi.Gen2Rx(adc_rate=adc, ntaps=ntaps, fixed_q=fixed_q)
    return _RX[key]


def oracle_for(adc, ntaps=25):
    from oracle.pyoracle import Oracle
    if (adc, ntaps) not in _OR:
        _OR[adc, ntaps] = Oracle(adc_rate=adc, ntaps=ntaps)
    return _OR[adc, ntaps]


def _assert_same(got, ref, what=""):
    bad = records_equal(got, ref)
    assert not bad, "%s fields differ: %s" % (what, bad)


@pytest.mark.parametrize("case", rate_cases(), ids=[c[0] for c in rate_cases()])
def test_rate_parity_with_reference_and_restatement(ref_rates, case):
    key, adc, ntaps, kw = case
    cap = rate_capture(adc, kw)
    iq = cap["iq"].numpy()
    recs, counts = rx_for(adc, ntaps, kw.get("fixed_q", 0)).decode_capture_host(iq, cap["segments"], max_windows=4)
    assert counts.tolist() == ref_rates[key + "_counts"].tolist()
    _assert_same(recs, ref_rates[key + "_records"], key + " vs reference")
    orecs, ocounts, _ = oracle_for(adc, ntaps).decode_segments(iq, cap["segments"], max_per_seg=4)
    assert counts.tolist() == ocounts.tolist()
    _assert_same(recs, orecs, key + " vs restatement")


def _kernel_names(fn):
    """names of the receive-chain kernels fn() launched (torch.profiler, CUDA activity only)"""
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


def _expected_kernel(adc, ntaps):
    if ntaps == 25 and adc in (R12, 2_000_000):
        return "rx_pack_kernel"
    return "rx_fused_split_kernel" if adc <= 2_400_000 else "rx_fused_kernel"


@pytest.mark.parametrize("adc,ntaps", RATES + [(2_000_000, 25)])
def test_kernel_chosen_per_rate(adc, ntaps):
    """which capture kernel decodes each rate: a change of the choice (pack_ok, fast_path_ok) would otherwise quietly turn
    a packed-kernel test into a split-kernel one"""
    cap = rate_capture(adc, {})
    rx = rx_for(adc, ntaps)
    names = _kernel_names(lambda: rx.decode_capture_host(cap["iq"].numpy(), cap["segments"], max_windows=4))
    assert names == {_expected_kernel(adc, ntaps)}, (adc, ntaps, names)


# ------------------------------------------------------------------ the packed kernel at 1.2 MS/s
@pytest.mark.parametrize("g", [1, 3, 7, 8])
def test_pack_kernel_at_1_2_msps_segments_per_cta(g, monkeypatch):
    """forced segments per CTA, ragged lengths (windows cut mid-way), odd offsets, a last CTA that is not full"""
    from gen2_uhf_rfid_reader_b200 import capi
    monkeypatch.setenv("RFID_B200_PACK_G", str(g))
    rxg = capi.Gen2Rx(adc_rate=R12)
    cap = synth.make_capture(23, seed=91, adc_rate=R12)
    iq = cap["iq"].numpy()
    segs = cap["segments"].copy()
    rng = np.random.default_rng(g)
    segs["length"] = (segs["length"] - rng.integers(0, 5400, size=segs.size)).astype(np.uint32)
    segs["offset"] = segs["offset"] + rng.integers(0, 3, size=segs.size).astype(np.uint64)
    names = _kernel_names(lambda: rxg.decode_capture_host(iq, segs, max_windows=4))
    assert names == {"rx_pack_kernel"}
    recs, counts = rxg.decode_capture_host(iq, segs, max_windows=4)
    orecs, ocounts, _ = oracle_for(R12).decode_segments(iq, segs, max_per_seg=4)
    assert counts.tolist() == ocounts.tolist() and counts.sum() >= 23
    _assert_same(recs, orecs, "1.2 MS/s G=%d" % g)


def _long_segments():
    """one segment = eight inventory rounds back to back: 16,281 decimated samples, nearly four trips around
    the 4096-sample history, 14-16 windows"""
    cap = synth.make_capture(24, seed=203, adc_rate=R12)
    segs = cap["segments"][::8].copy()
    segs["length"] = (8 * cap["segments"]["length"][0]).astype(np.uint32)
    return cap["iq"].numpy(), segs


@pytest.mark.parametrize("g", [0, 8])
def test_pack_kernel_at_1_2_msps_long_segments(g, monkeypatch):
    from gen2_uhf_rfid_reader_b200 import capi
    if g:
        monkeypatch.setenv("RFID_B200_PACK_G", str(g))
    rxg = capi.Gen2Rx(adc_rate=R12)
    iq, segs = _long_segments()
    recs, counts = rxg.decode_capture_host(iq, segs, max_windows=16)
    orecs, ocounts, _ = oracle_for(R12).decode_segments(iq, segs, max_per_seg=16)
    assert counts.tolist() == ocounts.tolist() and int(counts.max()) >= 12
    _assert_same(recs, orecs, "1.2 MS/s long segments, G=%d" % g)


def test_split_kernel_at_1_2_msps_on_the_same_inputs(monkeypatch):
    """RFID_B200_KERNEL=split on the packed kernel's inputs: ragged and long segments"""
    from gen2_uhf_rfid_reader_b200 import capi
    monkeypatch.setenv("RFID_B200_KERNEL", "split")
    rxs = capi.Gen2Rx(adc_rate=R12)
    cap = synth.make_capture(23, seed=91, adc_rate=R12)
    iq = cap["iq"].numpy()
    segs = cap["segments"].copy()
    rng = np.random.default_rng(3)
    segs["length"] = (segs["length"] - rng.integers(0, 5400, size=segs.size)).astype(np.uint32)
    segs["offset"] = segs["offset"] + rng.integers(0, 3, size=segs.size).astype(np.uint64)
    names = _kernel_names(lambda: rxs.decode_capture_host(iq, segs, max_windows=4))
    assert names == {"rx_fused_split_kernel"}
    recs, counts = rxs.decode_capture_host(iq, segs, max_windows=4)
    orecs, ocounts, _ = oracle_for(R12).decode_segments(iq, segs, max_per_seg=4)
    assert counts.tolist() == ocounts.tolist()
    _assert_same(recs, orecs, "1.2 MS/s split")
    iq, segs = _long_segments()
    recs, counts = rxs.decode_capture_host(iq, segs, max_windows=16)
    orecs, ocounts, _ = oracle_for(R12).decode_segments(iq, segs, max_per_seg=16)
    assert counts.tolist() == ocounts.tolist()
    _assert_same(recs, orecs, "1.2 MS/s split, long segments")


def test_pack_kernel_at_1_2_msps_window_tap():
    """the ungated windows (y - DC) the packed kernel decodes, byte for byte against the restatement's gate (the kernel
    is chosen from the configuration alone, which test_kernel_chosen_per_rate checks)"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    dev = torch.device("cuda:0")
    rx = rx_for(R12)
    iq_h, segs = _long_segments()
    n = int(segs["length"][0])
    x = iq_h[int(segs["offset"][0]):int(segs["offset"][0]) + n]
    iq = torch.from_numpy(x.copy()).to(dev)
    dsegs = capi.segments_to_device(abi.make_segments([0], [n]), dev)
    tap = torch.zeros((32, rx.len_epc), dtype=torch.complex64, device=dev)
    rx.set_window_tap(tap)
    try:
        res, cnt = rx.decode_capture(iq, dsegs, max_windows=32)
        torch.cuda.synchronize()
    finally:
        rx.set_window_tap(None)
    o = oracle_for(R12)
    g = o.gate(o.mf(x), max_windows=32, want_windows=True)
    k = int(cnt.cpu()[0])
    assert k == min(g["n"], 32) and k >= 12
    t = tap.cpu().numpy()
    for j in range(k):
        L = rx.len_epc if j & 1 else rx.len_rn16
        assert t[j, :L].tobytes() == g["windows"][j, :L].tobytes(), j


# ------------------------------------------------------------------ block mode (GNU Radio drop-in calls)
@pytest.mark.parametrize("adc", [R12, 2_400_000])
def test_block_mode_at_other_rates(adc):
    """mf_work in arbitrary chunks, gate_work in chunks, decoder_work on each window: against the restatement's matched
    filter, gate and window decoder"""
    from gen2_uhf_rfid_reader_b200 import capi
    o = oracle_for(adc)
    cap = synth.make_capture(6, seed=17, adc_rate=adc)
    x = cap["iq"].numpy()
    n = x.size - x.size % 5
    y_ref = o.mf(x[:n])
    rxm = capi.Gen2Rx(adc_rate=adc)
    chunks, pos = [], 0
    for sz in (1, 4, 5, 4096, 7777, 33333, n):
        if pos >= n:
            break
        chunks.append(rxm.mf_work(x[pos:min(n, pos + sz)]))
        pos = min(n, pos + sz)
    y = np.concatenate(chunks)
    assert y.size == n // 5 and y.tobytes() == y_ref.tobytes()

    g = o.gate(y_ref, want_windows=True)
    assert g["n"] >= 10
    rxg = capi.Gen2Rx(adc_rate=adc)
    pos, cur, seek, wins, it = 0, [], 1, [], 0
    sizes = [257, 4096, 1000, 8192]
    while pos < y_ref.size:
        r = rxg.gate_work(y_ref[pos:pos + sizes[it % 4]], seek=seek)
        it += 1
        seek = 0
        pos += r["consumed"]
        if r["written"]:
            cur.append(r["out"])
        if r["closed"]:
            wins.append(np.concatenate(cur))
            cur = []
            seek = 2 if (len(wins) & 1) else 1   # ACK -> SEEK_EPC, Query -> SEEK_RN16 (reader_impl.cc:262,296)
    assert len(wins) == g["n"]
    for k, w in enumerate(wins):
        kind = k & 1
        Lw = rxg.len_epc if kind else rxg.len_rn16
        assert w.size == Lw and w.tobytes() == g["windows"][k, :Lw].tobytes(), k
        rec, bits = rxg.decoder_work(kind, w)
        ref = o.decode_window(kind, w)
        for f in ("sync_index", "score", "h_re", "h_im", "T", "crc_ok", "tag_id", "bits", "kind", "length"):
            assert rec[f].tobytes() == ref[f].tobytes(), (adc, k, f)
        assert np.array_equal(bits, np.unpackbits(ref["bits"])[:bits.size].astype(np.float32))
