"""Capture mode: reply energy, decision SNR and slot outcome of every stored window (rfid_b200_window_quality).

CPU: the numpy restatement (quality_model.py) on the oracle's gate windows and records samples where the decoder samples,
sorts the simulator's slots by their number of replies and the reference recording's windows by whether the tag
answered, and keeps a tail of one symbol at every well-defined rate.  GPU: the device records equal the restatement's
bit for bit behind every kernel family that writes the window tap, and the outcomes of the closed-loop simulator's slots
match its truth.
"""
import ctypes as C

import numpy as np
import pytest

import quality_model as qm
import rate_rule
import segmenter_model as sm
from gen2_uhf_rfid_reader_b200 import abi, synth

Q4 = dict(seed=94, fixed_q=4, n_tags=8)


def _confusion(n_replies, outcome):
    """rows: 0, 1, >= 2 replies; columns: EMPTY, SINGLE, COLLISION"""
    m = np.zeros((3, 3), dtype=int)
    for r, o in zip(np.minimum(n_replies, 2), outcome):
        m[r, o] += 1
    return m


def _check_floors(m):
    """every empty and every single slot right, at least 95 % of the collided slots"""
    assert m[0, 0] == m[0].sum() and m[1, 1] == m[1].sum(), m
    assert m[2, 2] >= 0.95 * m[2].sum(), m


def _check_recording(recs, q):
    """every RN16 window SINGLE; every EPC window whose CRC passes SINGLE; the one whose CRC fails (the tag had stopped
    waiting for its ACK, 1738.5 us after its RN16) EMPTY"""
    rn, ep = recs["kind"] == abi.RN16, recs["kind"] == abi.EPC
    ok = recs["crc_ok"] == 1
    assert rn.sum() == ep.sum() == 71 and (ep & ~ok).sum() == 1
    assert (q["outcome"][rn] == abi.SLOT_SINGLE).all()
    assert (q["outcome"][ep & ok] == abi.SLOT_SINGLE).all()
    bad = q[ep & ~ok][0]
    assert bad["outcome"] == abi.SLOT_EMPTY and 10 * np.log10(bad["energy"]) < 1.0
    assert (q["n_decisions"] == np.where(rn, 16, 128)).all()


@pytest.fixture(scope="module")
def rec_windows(oracle, cfg1_iq):
    return qm.oracle_windows(oracle, cfg1_iq, abi.make_segments([0], [cfg1_iq.size]), 160)


@pytest.fixture(scope="module")
def q4_windows(oracle):
    cap = synth.make_capture(1024, device="cpu", **Q4)
    return cap, qm.oracle_windows(oracle, cap["iq"].numpy(), cap["segments"], 2)


# ------------------------------------------------------------------ CPU: the rule
def test_projections_reproduce_the_decoders_bits(rec_windows, q4_windows, oracle):
    """the signs of the model's projections are the oracle's RN16 and EPC bits, window by window"""
    n_f = oracle.cfg.n_tag_bit_f
    (_, (w2, r2, c2)) = q4_windows
    w1, r1, c1 = rec_windows
    n = 0
    for w, r, c in ((w1, r1, c1), (w2, r2, c2)):
        for s in range(c.size):
            for k in range(min(int(c[s]), r.shape[1])):
                _, bits = qm.decisions(w[s, k], r[s, k], n_f)
                nb = 2 if int(r[s, k]["kind"]) == abi.RN16 else 16
                assert bits.tobytes() == r[s, k]["bits"][:nb].tobytes(), (s, k)
                n += 1
    assert n == 142 + 2048


def test_outcomes_on_the_recording(rec_windows):
    w, r, c = rec_windows
    q = qm.quality(w, r, c)[0, :c[0]]
    _check_recording(r[0, :c[0]], q)


def test_confusion_matrix_on_the_q4_simulation(q4_windows):
    """synth.make_capture(1024, seed=94, fixed_q=4, n_tags=8) at the default noise, default thresholds: every empty and
    single slot right, 90 of 91 collisions (the other has a decision SNR of 11.0 dB)"""
    cap, (w, r, c) = q4_windows
    q = qm.quality(w, r, c)
    m = _confusion(cap["truth"]["n_replies"], q["outcome"][:, 0])
    assert m.tolist() == [[615, 0, 0], [0, 318, 0], [0, 1, 90]], m
    _check_floors(m)
    # the open-loop simulator ACKs the strongest tag of every slot that has one, so every EPC that passes is a reply
    ok = r[:, 1]["crc_ok"] == 1
    assert ok.sum() == 409 and (q["outcome"][ok, 1] == abi.SLOT_SINGLE).all()


def test_noise_reference_holds_no_rn16_reply_at_every_well_defined_rate():
    """at every sync index the preamble search can return, an RN16 window's noise reference holds at least one symbol
    (n_tag_bit_i samples) that lie before the reply or after it, and the reply span at least 116 samples (decimation 5,
    every 7th well-defined rate of the 1 kHz grid from 1 to 8 MS/s); an EPC window's reference holds one symbol, though
    for a slow tag clock part of it can lie in the reply's end"""
    grid = rate_rule.GRID[rate_rule.well_defined(rate_rule.GRID)][::7]
    for adc in list(grid) + [1_000_000, 2_000_000, 8_000_000]:
        n_i = qm.derived(int(adc))[0]
        reply, noise, clean = qm.noise_extents(int(adc))
        assert clean[0] >= n_i and noise[1] >= n_i and min(reply) >= 116, (adc, reply, noise, clean)


@pytest.mark.parametrize("d", [0, 3, 6, 9])
def test_outcomes_on_the_recording_with_late_replies(oracle, cfg1_iq, d):
    """the recording's windows opened d samples early, so that every reply sits d samples later in its window (sync
    index 4-6 + d, as for tags with a longer T1): every RN16 window that decodes as before is SINGLE, every EPC window
    whose CRC passes SINGLE, the one whose CRC fails EMPTY"""
    w, r, c = qm.early_windows(oracle, cfg1_iq, d)
    q = qm.quality(w, r, c)[0]
    r = r[0]
    base = qm.early_windows(oracle, cfg1_iq, 0)[1][0]
    same = (r["bits"] == base["bits"]).all(axis=1)
    assert same.sum() >= 141 and np.median(r["sync_index"]) == np.median(base["sync_index"]) + d
    rn, ep, ok = r["kind"] == abi.RN16, r["kind"] == abi.EPC, r["crc_ok"] == 1
    assert (q["outcome"][rn & same] == abi.SLOT_SINGLE).all()
    assert (q["outcome"][ep & ok] == abi.SLOT_SINGLE).all() and (ep & ok).sum() == 70
    assert (q["outcome"][ep & ~ok] == abi.SLOT_EMPTY).all()


@pytest.mark.parametrize("dt", [10.0, 20.0])
def test_confusion_matrix_with_a_later_tag_reply(oracle, monkeypatch, dt):
    """the Q = 4 simulation with every tag's T1 dt microseconds longer (replies 4 and 8 samples later in their windows):
    the same confusion matrix as at the nominal T1"""
    monkeypatch.setattr(synth, "T1_TAG_US", synth.T1_TAG_US + dt)
    cap = synth.make_capture(1024, device="cpu", **Q4)
    w, r, c = qm.oracle_windows(oracle, cap["iq"].numpy(), cap["segments"], 2)
    assert r[cap["truth"]["n_replies"] == 1, 0]["sync_index"].min() >= 4 + int(dt * 0.4)
    q = qm.quality(w, r, c)
    m = _confusion(cap["truth"]["n_replies"], q["outcome"][:, 0])
    assert m.tolist() == [[615, 0, 0], [0, 318, 0], [0, 1, 90]], m
    ok = r[:, 1]["crc_ok"] == 1
    assert (q["outcome"][ok, 1] == abi.SLOT_SINGLE).all()


def test_defaults_layouts_and_null_context():
    from gen2_uhf_rfid_reader_b200 import capi
    qp = capi.default_quality_params()
    assert (qp.empty_db, qp.single_snr_db) == (np.float32(qm.DEFAULT_EMPTY_DB), np.float32(qm.DEFAULT_SINGLE_SNR_DB))
    assert list(qp.reserved) == [0] * 6
    assert C.sizeof(abi.QualityParams) == 32 and C.sizeof(abi.Quality) == 16
    assert abi.QUALITY_DTYPE == qm.QUALITY_DTYPE
    for name, _ in abi.Quality._fields_:
        assert getattr(abi.Quality, name).offset == abi.QUALITY_DTYPE.fields[name][1]
    assert (abi.SLOT_EMPTY, abi.SLOT_SINGLE, abi.SLOT_COLLISION) == (qm.EMPTY, qm.SINGLE, qm.COLLISION)
    L = capi.load_library()
    buf = np.zeros(64, dtype=np.float32)
    assert L.rfid_b200_window_quality(None, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, 1, 1, None,
                                      buf.ctypes.data, None) == abi.EINVAL
    L.rfid_b200_default_quality_params(None)   # tolerated


def test_slot_table_and_summary():
    from gen2_uhf_rfid_reader_b200 import capi
    recs = np.zeros((3, 2), dtype=abi.RESULT_DTYPE)
    recs["kind"][:, 1] = abi.EPC
    recs["crc_ok"][:, 1] = [1, 0, 1]
    recs["tag_id"][:, 1] = [0x27, 5, 0x28]
    q = np.zeros((3, 2), dtype=abi.QUALITY_DTYPE)
    q["energy"], q["snr"] = 100.0, 10.0
    q["outcome"][:, 0] = [abi.SLOT_SINGLE, abi.SLOT_COLLISION, abi.SLOT_EMPTY]
    q["outcome"][:, 1] = abi.SLOT_SINGLE
    counts = np.array([2, 2, 1])
    t = capi.slot_table(recs, counts, q)
    assert t["rn16_outcome"].tolist() == [1, 2, 0] and t["epc_outcome"].tolist() == [1, 1, -1]
    assert t["tag_id"].tolist() == [0x27, 5, -1] and t["crc_ok"].tolist() == [1, 0, -1]
    assert t["rn16_energy_db"].tolist() == [20.0] * 3 and np.isnan(t["epc_snr_db"][2])
    s = capi.inventory_summary(recs, counts, q)
    assert s == {"slots": 3, "empty": 1, "single": 1, "collision": 1, "single_epc_ok": 1}


# ------------------------------------------------------------------ GPU
def _rx(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx(**kw)


def _device(rx, iq, segs, max_windows, params=None, sentinel=False):
    """decode_capture with the tap, then window_quality: host (windows, recs, counts, quality).  iq, segs: CUDA tensors.
    sentinel: fill the quality buffer with 0xAB bytes first"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    nseg = segs.numel() // 16
    tap = torch.zeros(nseg * max_windows * rx.len_epc, dtype=torch.complex64, device="cuda")
    rx.set_window_tap(tap)
    try:
        res, cnt = rx.decode_capture(iq, segs, max_windows=max_windows)
    finally:
        rx.set_window_tap(None)
    quality = torch.full((nseg * max_windows, 16), 0xAB if sentinel else 0, dtype=torch.uint8, device="cuda")
    rx.window_quality(tap, res, cnt, max_windows, params=params, quality=quality)
    torch.cuda.synchronize()
    recs, counts = capi.results_to_numpy(res, cnt, max_windows)
    q, _ = capi.quality_to_numpy(quality, cnt, max_windows)
    return tap.cpu().numpy().reshape(nseg, max_windows, rx.len_epc), recs, counts, q


def _same_as_model(rx, dev, adc=2_000_000, **kw):
    """the device records equal the restatement's on the tap, and the signs of the projections of the tap's samples are
    the bits the device decoder stored (the tap holds what the decoder read)"""
    w, recs, counts, q = dev
    want = qm.quality(w, recs, counts, adc_rate=adc, **kw)
    stored = np.arange(recs.shape[1])[None, :] < np.minimum(counts, recs.shape[1])[:, None]
    assert q[stored].tobytes() == want[stored].tobytes()
    n_f = qm.derived(adc)[1]
    for s, k in zip(*np.nonzero(stored)):
        nb = 2 if int(recs[s, k]["kind"]) == abi.RN16 else 16
        assert qm.decisions(w[s, k], recs[s, k], n_f)[1].tobytes() == recs[s, k]["bits"][:nb].tobytes(), (s, k)
    return q


def _cuda(x, segs):
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    return torch.from_numpy(np.ascontiguousarray(x)).cuda(), capi.segments_to_device(segs, "cuda")


@pytest.fixture(scope="module")
def rx():
    return _rx()


@pytest.mark.gpu
def test_device_on_the_recording(rx, cfg1_iq):
    """whole and as the segmenter's segments: the restatement bit for bit, and the recording's outcomes"""
    whole = abi.make_segments([0], [cfg1_iq.size])
    dev = _device(rx, *_cuda(cfg1_iq, whole), 160)
    q = _same_as_model(rx, dev)
    recs, counts = dev[1], dev[2]
    assert counts.tolist() == [142]
    _check_recording(recs[0, :142], q[0, :142])
    segs, _ = sm.segment_table(cfg1_iq)
    segs = abi.make_segments([o for o, _ in segs], [n for _, n in segs])
    dev = _device(rx, *_cuda(cfg1_iq, segs), 4)
    q = _same_as_model(rx, dev)
    recs, counts = dev[1], dev[2]
    flat = lambda a: np.concatenate([a[s, :min(counts[s], 4)] for s in range(counts.size)])   # noqa: E731
    _check_recording(flat(recs), flat(q))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["q4", "noisy", "sc16", "params"])
def test_device_on_synthetic_captures(rx, case):
    """Q = 4 with 8 tags, heavy noise, an sc16 capture (decoded as its conversion; the tap is float2 either way), other
    thresholds"""
    import torch
    noise = dict(noise_sigma=0.02) if case == "noisy" else {}
    cap = synth.make_capture(512, device="cuda", **Q4, **noise)
    segs = cap["segments"]
    x = cap["iq"].cpu().numpy()
    params, kw = None, {}
    if case == "params":
        from gen2_uhf_rfid_reader_b200 import capi
        params, kw = capi.default_quality_params(empty_db=-3.0, single_snr_db=25.0), dict(empty_db=-3.0, single_snr_db=25.0)
    if case == "sc16":
        from test_sc16 import SCALES, quantise
        q16 = quantise(x, SCALES[0])
        iq16, dsegs = _cuda(q16, segs)
        nseg = len(segs)
        tap = torch.zeros(nseg * 2 * rx.len_epc, dtype=torch.complex64, device="cuda")
        rx.set_window_tap(tap)
        try:
            res, cnt = rx.decode_capture(iq16, dsegs, max_windows=2, scale=SCALES[0])
        finally:
            rx.set_window_tap(None)
        r2, c2, quality = rx.decode_capture_quality(iq16, dsegs, max_windows=2, scale=SCALES[0])
        from gen2_uhf_rfid_reader_b200 import capi
        recs, counts = capi.results_to_numpy(res, cnt, 2)
        q, _ = capi.quality_to_numpy(quality, c2, 2)
        assert capi.results_to_numpy(r2, c2, 2)[0].tobytes() == recs.tobytes()
        dev = (tap.cpu().numpy().reshape(nseg, 2, rx.len_epc), recs, counts, q)
    else:
        dev = _device(rx, *_cuda(x, segs), 2, params=params)
    q = _same_as_model(rx, dev, **kw)
    if case == "q4":
        m = _confusion(cap["truth"]["n_replies"], q["outcome"][:, 0])
        _check_floors(m)
    assert (dev[2] == 2).all()


FAMILIES = [(2_000_000, None), (1_200_000, None), (2_000_000, "split"), (4_000_000, None), (8_000_000, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("adc,kernel", FAMILIES, ids=["pack-2M", "pack-1.2M", "split-2M", "fused-4M", "fused-8M"])
def test_device_behind_every_kernel_family(adc, kernel, monkeypatch):
    """rx_pack_kernel at 2 and 1.2 MS/s, the split kernel (RFID_B200_KERNEL=split) and rx_fused_kernel at 4 and 8 MS/s
    write the tap the quality kernel reads; the records equal the restatement's"""
    if kernel:
        monkeypatch.setenv("RFID_B200_KERNEL", kernel)
    rxk = _rx(adc_rate=adc, ntaps=max(12, adc // 80000), fixed_q=2)
    cap = synth.make_capture(96, adc_rate=adc, seed=31, fixed_q=2, n_tags=4, device="cuda")
    dev = _device(rxk, *_cuda(cap["iq"].cpu().numpy(), cap["segments"]), 3)
    _same_as_model(rxk, dev, adc=adc)
    assert (dev[2] >= 2).all()
    m = _confusion(cap["truth"]["n_replies"], dev[3]["outcome"][:, 0])
    assert m[0, 0] == m[0].sum() and m[1, 1] == m[1].sum(), m


@pytest.mark.gpu
@pytest.mark.parametrize("q,tags", [(2, 4), (4, 8)], ids=["q2-4tags", "q4-8tags"])
def test_closed_loop_simulator_against_truth(q, tags):
    """rfid_b200_sim_capture, closed loop: outcomes against the simulator's n_replies with the floors of the CPU test;
    every EPC that passes its CRC is SINGLE; the first slots equal the restatement bit for bit"""
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = _rx(fixed_q=q)
    cap = rxq.sim_capture(capi.default_sim(n_tags=tags, closed_loop=1, seed=700 + q), 2048)
    res, cnt, quality = rxq.decode_capture_quality(cap["iq"], cap["segs"], max_windows=2)
    recs, counts = capi.results_to_numpy(res, cnt, 2)
    qq, _ = capi.quality_to_numpy(quality, cnt, 2)
    truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
    assert (counts == 2).all()
    m = _confusion(truth["n_replies"], qq["outcome"][:, 0])
    _check_floors(m)
    assert m[2].sum() > 0 and m[0].sum() > 0
    ok = recs[:, 1]["crc_ok"] == 1
    assert ok.sum() > 0 and (qq["outcome"][ok, 1] == abi.SLOT_SINGLE).all()
    s = capi.inventory_summary(recs, counts, qq)
    assert (s["empty"], s["single"], s["collision"]) == tuple(m.sum(axis=0)) and s["single_epc_ok"] <= ok.sum()
    k = 64
    dev = _device(rxq, cap["iq"][:k * cap["segment_len"]], cap["segs"][:k], 2)
    want = _same_as_model(rxq, dev)
    assert want.tobytes() == qq[:k].tobytes()


@pytest.mark.gpu
def test_device_writes_only_stored_records(rx, cfg1_iq):
    """segments with more windows than max_windows, with none, and with fewer than max_windows: nothing is written beyond
    the stored records"""
    one = int(sm.segment_table(cfg1_iq)[0][1][0])       # the second segment of the segmenter's table ...
    segs = abi.make_segments([0, 0, 1000, 5, one], [cfg1_iq.size, 300000, 40, 0, 8000])   # ... cut to its RN16 window
    w, recs, counts, q = _device(rx, *_cuda(cfg1_iq, segs), 3, sentinel=True)
    assert counts.tolist()[:4] == [142, counts[1], 0, 0] and counts[1] > 3 and counts[4] == 1
    raw = q.view(np.uint8).reshape(5, 3, 16)
    assert (raw[2:4] == 0xAB).all() and (raw[4, 1:] == 0xAB).all()
    assert (raw[:2] != 0xAB).any(axis=2).all() and (raw[4, 0] != 0xAB).any()
    _same_as_model(rx, (w, recs, counts, q))


@pytest.mark.gpu
def test_window_quality_argument_checks(rx):
    """a NULL window buffer (or any NULL pointer), non-finite thresholds, negative counts: RFID_B200_EINVAL"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    tap = torch.zeros(2 * rx.len_epc, dtype=torch.complex64, device="cuda")
    res = torch.zeros((2, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.zeros((2, 16), dtype=torch.uint8, device="cuda")

    def call(w=tap.data_ptr(), r=res.data_ptr(), c=cnt.data_ptr(), o=out.data_ptr(), n=1, m=2, p=None):
        return L.rfid_b200_window_quality(rx.h, w, r, c, n, m, p, o, None)

    assert call() == abi.OK and call(n=0) == abi.OK and call(m=0) == abi.OK
    for kw in (dict(w=None), dict(r=None), dict(c=None), dict(o=None), dict(n=-1), dict(m=-1)):
        assert call(**kw) == abi.EINVAL, kw
    for bad in (float("nan"), float("inf"), float("-inf")):
        for f in ("empty_db", "single_snr_db"):
            assert call(p=C.byref(capi.default_quality_params(**{f: bad}))) == abi.EINVAL, (f, bad)
            with pytest.raises(capi.RfidB200Error):
                rx.window_quality(tap, res, cnt, 2, params=capi.default_quality_params(**{f: bad}))
    torch.cuda.synchronize()
    assert (out == 0).all()
