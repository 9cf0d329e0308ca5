"""Capture mode: recovery of EPC replies that fail their CRC (rfid_b200_recover_epc).

CPU: the numpy restatement (recover_model.py) tests candidates through a syndrome that equals the bit rule's; on the
oracle's windows of the reference recording and of a weak simulated tag it recovers every window whose sign errors are a
candidate (or calls it ambiguous) and never one that differs from the truth; empty slots are not attempted; random
windows are recovered no more often than the false-accept bound allows.  GPU: the device records equal the
restatement's bit for bit behind every kernel family that writes the window tap, and the closed-loop simulator's
recovered EPCs equal its truth.
"""
import ctypes as C

import numpy as np
import pytest

import quality_model as qm
import recover_model as rm
from gen2_uhf_rfid_reader_b200 import abi, synth

WEAK = dict(seed=77)                                    # one tag
Q4_WEAK = dict(seed=78, fixed_q=4, n_tags=8, tag_gain=0.004)


def _windows(oracle, cap, max_windows=2):
    return qm.oracle_windows(oracle, cap["iq"].numpy(), cap["segments"], max_windows)


@pytest.fixture(scope="module")
def rec_windows(oracle, cfg1_iq):
    return qm.oracle_windows(oracle, cfg1_iq, abi.make_segments([0], [cfg1_iq.size]), 160)


# ------------------------------------------------------------------ CPU: the rule
def test_syndrome_form_against_the_bit_rule():
    """the linear syndrome equals the CRC-16 + PC-length rule on every single sign flip of valid frames and on random
    flip sets of random words, and the verdict (syndrome 0) is the rule's"""
    from gen2_uhf_rfid_reader_b200 import synth as sy
    rng = np.random.default_rng(5)
    frames = sy.make_epc_frames(rng.integers(0, 256, size=(4, 12)).astype(np.uint8))
    for f in frames:
        assert rm.syndrome(f) == 0 and rm.syndrome_direct(f) == 0
        b = np.unpackbits(f)
        for j in range(128):   # one sign flip: bits j and j + 1
            x = b.copy()
            x[j] ^= 1
            if j < 127:
                x[j + 1] ^= 1
            w = np.packbits(x)
            assert rm.syndrome(w) == rm.syndrome_direct(w) == rm.SIGN_COL[j] != 0, j
    for _ in range(400):
        w = rng.integers(0, 256, size=16).astype(np.uint8)
        F = rng.choice(128, size=rng.integers(1, 7), replace=False)
        x = np.unpackbits(w)
        for j in F:
            x[j] ^= 1
            if j < 127:
                x[j + 1] ^= 1
        v = np.packbits(x)
        assert rm.syndrome(v) == rm.syndrome_direct(v) == rm.syndrome(w) ^ np.bitwise_xor.reduce(rm.SIGN_COL[F])
        ok = (sy.crc16_gen2(bytes(v[:14])) == int.from_bytes(bytes(v[14:16]), "big")) and (v[0] >> 3) == 0b00110
        assert ok == (rm.syndrome(v) == 0)
    assert rm.n_candidates() == 793 and abs(rm.false_accept_bound() - 3.78e-4) < 1e-6


def test_recording(rec_windows):
    """71 RN16 windows NOT_EPC, 70 EPC windows CRC_OK; the one that fails (acknowledged 1738.5 us after its RN16, so
    the tag no longer answered: energy -0.2 dB) has a decision SNR of 2.4 dB, that of pure noise, and is SKIPPED"""
    w, r, c = rec_windows
    q = qm.quality(w, r, c)
    fx = rm.recover(w, r, c, q)[0, :c[0]]
    st = fx["status"]
    assert (st == rm.NOT_EPC).sum() == 71 and (st == rm.CRC_OK).sum() == 70 and (st == rm.SKIPPED).sum() == 1
    bad = np.nonzero(st == rm.SKIPPED)[0][0]
    assert r[0, bad]["crc_ok"] == 0 and round(float(10 * np.log10(q[0, bad]["snr"])), 1) == 2.4
    assert (fx["bits"] == r[0, :c[0]]["bits"]).all() and np.isnan(fx["cost"]).all()


@pytest.mark.parametrize("g,before,after", [(0.004, 540, 595), (0.003, 388, 502)])
def test_weak_tag(oracle, g, before, after):
    """synth.make_capture(600, seed=77, tag_gain=g), one tag: every window whose sign errors E number 1..W, lie among
    the P least reliable and pass the SNR gate is RECOVERED with the true bits, or AMBIGUOUS; no RECOVERED window
    differs from the truth; the EPC reads rise from `before` to `after`, and the READER_STATS count them"""
    from gen2_uhf_rfid_reader_b200 import capi
    cap = synth.make_capture(600, device="cpu", tag_gain=g, **WEAK)
    w, r, c = _windows(oracle, cap)
    q = qm.quality(w, r, c)
    fx = rm.recover(w, r, c, q)
    truth = cap["truth"]["epc"]
    n_f, mr = oracle.cfg.n_tag_bit_f, rm.snr_ratio()
    st = fx[:, 1]["status"]
    eligible = 0
    for s in range(c.size):
        if r[s, 1]["crc_ok"] == 1:
            continue
        rr = rm.epc_projections(w[s, 1], r[s, 1], n_f, oracle.cfg.len_epc)
        E = rm.sign_errors(rr, truth[s])
        least = np.argsort(np.abs(rr), kind="stable")[:rm.DEFAULT_P]
        if 1 <= E.size <= rm.DEFAULT_W and np.isin(E, least).all() and q[s, 1]["snr"] >= mr:
            eligible += 1
            assert st[s] in (rm.RECOVERED, rm.AMBIGUOUS), s
        if st[s] == rm.RECOVERED:
            assert fx[s, 1]["bits"].tobytes() == truth[s].tobytes(), s
            assert synth.crc16_gen2(bytes(fx[s, 1]["bits"][:14])) == int.from_bytes(bytes(fx[s, 1]["bits"][14:]), "big")
    n_rec = int((st == rm.RECOVERED).sum())
    assert eligible > 0 and n_rec >= eligible - int((st == rm.AMBIGUOUS).sum())
    assert (r[:, 1]["crc_ok"] == 1).sum() == before
    fixed = capi.apply_fixes(r, c, fx)
    assert (fixed[:, 1]["crc_ok"] == 1).sum() == after == before + n_rec
    assert (fixed["tag_id"][:, 1][st == rm.RECOVERED] == 0x27).all()
    s0, s1 = oracle.reduce_stats(r, c, False), oracle.reduce_stats(fixed, c, False)
    assert s1.n_epc_correct == s0.n_epc_correct + n_rec
    assert s1.tag_map() == {0x27: after}


def test_empty_slots_are_not_attempted(oracle):
    """make_capture(1024, seed=78, fixed_q=4, n_tags=8, tag_gain=0.004): the EPC window of every empty slot is SKIPPED
    at the default min_snr_db (their decision SNR stays below 4.3 dB).  With the gate open (min_snr_db -100) every
    one of them is attempted; at most the false-accept bound's share may then be RECOVERED, and the count is pinned so
    that a change shows"""
    cap = synth.make_capture(1024, device="cpu", **Q4_WEAK)
    w, r, c = _windows(oracle, cap)
    q = qm.quality(w, r, c)
    empty = cap["truth"]["n_replies"] == 0
    assert empty.sum() == 612 and (c == 2).all()
    assert 10 * np.log10(q[empty, 1]["snr"].max()) < 4.3
    fx = rm.recover(w, r, c, q)
    assert (fx[empty, 1]["status"] == rm.SKIPPED).all()
    open_ = rm.recover(w[empty], r[empty], c[empty], q[empty], min_snr_db=-100.0)[:, 1]
    assert (open_["status"] != rm.SKIPPED).all()
    n_wrong = int((open_["status"] == rm.RECOVERED).sum())
    print("empty slots RECOVERED with the gate open: %d of %d" % (n_wrong, empty.sum()))
    assert n_wrong == 0


def test_false_accept_bound():
    """10^5 windows of Gaussian projections and random words (no true solution): the RECOVERED fraction is at most
    C * 2^-21 plus a 4-sigma binomial margin, at the default P and W"""
    rng = np.random.default_rng(2024)
    N = 100_000
    rho = np.abs(rng.standard_normal((N, 128)).astype(np.float32))
    bits = rng.integers(0, 256, size=(N, 16)).astype(np.uint8)
    n_pass = rm.n_pass_batch(rho, bits)
    p = rm.false_accept_bound()
    recovered = int((n_pass == 1).sum())
    print("random windows: %d of %d RECOVERED, %d AMBIGUOUS (bound %.1f)" % (recovered, N, int((n_pass >= 2).sum()),
                                                                          N * p))
    assert recovered <= N * p + 4 * np.sqrt(N * p * (1 - p))
    assert recovered > 0   # the bound is not vacuous: random words do pass now and then


def test_defaults_layouts_and_null_context():
    from gen2_uhf_rfid_reader_b200 import capi
    rp = capi.default_recover_params()
    assert (rp.positions, rp.max_flips, rp.min_snr_db) == (rm.DEFAULT_P, rm.DEFAULT_W, np.float32(rm.DEFAULT_MIN_SNR_DB))
    assert list(rp.reserved) == [0] * 5
    assert C.sizeof(abi.RecoverParams) == 32 and C.sizeof(abi.EpcFix) == 32
    assert abi.EPC_FIX_DTYPE == rm.EPC_FIX_DTYPE
    for name, _ in abi.EpcFix._fields_:
        assert getattr(abi.EpcFix, name).offset == abi.EPC_FIX_DTYPE.fields[name][1]
    assert (abi.FIX_CRC_OK, abi.FIX_RECOVERED, abi.FIX_AMBIGUOUS, abi.FIX_FAILED, abi.FIX_SKIPPED, abi.FIX_NOT_EPC) == \
        (rm.CRC_OK, rm.RECOVERED, rm.AMBIGUOUS, rm.FAILED, rm.SKIPPED, rm.NOT_EPC)
    assert "rfid_b200_recover_epc" in capi.EXPORTED_SYMBOLS and "rfid_b200_default_recover_params" in capi.EXPORTED_SYMBOLS
    L = capi.load_library()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    assert L.rfid_b200_recover_epc(None, p, p, p, p, 1, 1, None, p, None) == abi.EINVAL
    L.rfid_b200_default_recover_params(None)   # tolerated


def test_apply_fixes():
    """RECOVERED stored windows get the fix's bits, crc_ok 1 and tag_id = byte 13; nothing else changes"""
    from gen2_uhf_rfid_reader_b200 import capi
    recs = np.zeros((3, 2), dtype=abi.RESULT_DTYPE)
    recs["kind"][:, 1] = abi.EPC
    recs["tag_id"][:, 1] = 7
    fx = np.zeros((3, 2), dtype=abi.EPC_FIX_DTYPE)
    fx["status"][:, 1] = [abi.FIX_RECOVERED, abi.FIX_FAILED, abi.FIX_RECOVERED]
    fx["bits"][:, 1, 13] = 0x29
    fx["bits"][:, 1, 0] = 0x30
    counts = np.array([2, 2, 1])
    out = capi.apply_fixes(recs, counts, fx)
    assert out["crc_ok"][:, 1].tolist() == [1, 0, 0] and out["tag_id"][:, 1].tolist() == [0x29, 7, 7]
    assert out["bits"][0, 1].tobytes() == fx["bits"][0, 1].tobytes() and (out["bits"][1:] == 0).all()
    assert (recs["crc_ok"] == 0).all()   # a copy


# ------------------------------------------------------------------ GPU
def _rx(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx(**kw)


def _cuda(x, segs):
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    return torch.from_numpy(np.ascontiguousarray(x)).cuda(), capi.segments_to_device(segs, "cuda")


def _device(rx, iq, segs, max_windows, params=None, sentinel=False, scale=None):
    """decode_capture with the tap, window_quality, then recover_epc: host (windows, recs, counts, quality, fixes).
    Checks that the call leaves the records, counts and quality as they were.  sentinel: fill the fix buffer with 0xAB
    bytes first"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    nseg = segs.numel() // 16
    tap = torch.zeros(nseg * max_windows * rx.len_epc, dtype=torch.complex64, device="cuda")
    rx.set_window_tap(tap)
    try:
        kw = dict(scale=scale) if scale is not None else {}
        res, cnt = rx.decode_capture(iq, segs, max_windows=max_windows, **kw)
    finally:
        rx.set_window_tap(None)
    quality = rx.window_quality(tap, res, cnt, max_windows)
    before = (res.clone(), cnt.clone(), quality.clone())
    fixes = torch.full((nseg * max_windows, 32), 0xAB if sentinel else 0, dtype=torch.uint8, device="cuda")
    rx.recover_epc(tap, res, cnt, quality, max_windows, params=params, fixes=fixes)
    torch.cuda.synchronize()
    for a, b in zip(before, (res, cnt, quality)):
        assert torch.equal(a, b)
    recs, counts = capi.results_to_numpy(res, cnt, max_windows)
    q, _ = capi.quality_to_numpy(quality, cnt, max_windows)
    fx, _ = capi.fixes_to_numpy(fixes, cnt, max_windows)
    return tap.cpu().numpy().reshape(nseg, max_windows, rx.len_epc), recs, counts, q, fx


def _same_as_model(dev, adc=2_000_000, params=None):
    w, recs, counts, q, fx = dev
    kw = {}
    if params is not None:
        kw = dict(P=params.positions, W=params.max_flips, min_snr_db=params.min_snr_db)
    want = rm.recover(w, recs, counts, q, adc_rate=adc, **kw)
    stored = np.arange(recs.shape[1])[None, :] < np.minimum(counts, recs.shape[1])[:, None]
    assert fx[stored].tobytes() == want[stored].tobytes()
    return fx


def _no_wrong_recovery(fx, truth_epc):
    rec = fx[:, 1]["status"] == abi.FIX_RECOVERED
    assert (fx[rec, 1]["bits"] == truth_epc[rec]).all()
    return int(rec.sum())


@pytest.fixture(scope="module")
def rx():
    return _rx()


@pytest.mark.gpu
def test_device_on_the_recording(rx, cfg1_iq):
    dev = _device(rx, *_cuda(cfg1_iq, abi.make_segments([0], [cfg1_iq.size])), 160)
    fx = _same_as_model(dev)[0, :142]
    st = fx["status"]
    assert (st == abi.FIX_NOT_EPC).sum() == 71 and (st == abi.FIX_CRC_OK).sum() == 70 and (st == abi.FIX_SKIPPED).sum() == 1


FAMILIES = [(2_000_000, None), (1_200_000, None), (2_000_000, "split"), (4_000_000, None), (8_000_000, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("adc,kernel", FAMILIES, ids=["pack-2M", "pack-1.2M", "split-2M", "fused-4M", "fused-8M"])
def test_device_behind_every_kernel_family(adc, kernel, monkeypatch):
    """weak-tag captures decoded by rx_pack_kernel at 2 and 1.2 MS/s, the split kernel (RFID_B200_KERNEL=split) and
    rx_fused_kernel at 4 and 8 MS/s: the fixes equal the restatement's at the defaults and with the gate open; no
    RECOVERED window differs from the truth at the defaults.  The matched filter sums adc / 400 kHz samples per half
    symbol, so the gain scales as 1 / sqrt(adc) to keep the decisions as noisy as at 0.003 and 2 MS/s"""
    from gen2_uhf_rfid_reader_b200 import capi
    if kernel:
        monkeypatch.setenv("RFID_B200_KERNEL", kernel)
    rxk = _rx(adc_rate=adc, ntaps=max(12, adc // 80000))
    cap = synth.make_capture(128, adc_rate=adc, seed=31, tag_gain=0.003 * (2e6 / adc) ** 0.5, device="cuda")
    iq, segs = _cuda(cap["iq"].cpu().numpy(), cap["segments"])
    fx = _same_as_model(_device(rxk, iq, segs, 2), adc=adc)
    _no_wrong_recovery(fx, cap["truth"]["epc"])
    open_ = capi.default_recover_params(min_snr_db=-100.0)
    fx = _same_as_model(_device(rxk, iq, segs, 2, params=open_), adc=adc, params=open_)
    st = fx[:, 1]["status"]
    print("%s: %s" % (kernel or adc, np.bincount(st, minlength=6).tolist()))
    assert ((st >= abi.FIX_RECOVERED) & (st <= abi.FIX_FAILED)).sum() > 0 and (st == abi.FIX_SKIPPED).sum() == 0


@pytest.mark.gpu
def test_device_on_an_sc16_copy(rx):
    """the weak-tag capture quantised to sc16: decode_capture_recover equals the separate calls, and the restatement"""
    from gen2_uhf_rfid_reader_b200 import capi
    from test_sc16 import SCALES, quantise
    cap = synth.make_capture(256, device="cpu", tag_gain=0.003, **WEAK)
    q16 = quantise(cap["iq"].numpy(), SCALES[0])
    iq16, segs = _cuda(q16, cap["segments"])
    dev = _device(rx, iq16, segs, 2, scale=SCALES[0])
    fx = _same_as_model(dev)
    r2, c2, q2, f2 = rx.decode_capture_recover(iq16, segs, max_windows=2, scale=SCALES[0])
    assert capi.results_to_numpy(r2, c2, 2)[0].tobytes() == dev[1].tobytes()
    assert capi.quality_to_numpy(q2, c2, 2)[0].tobytes() == dev[3].tobytes()
    assert capi.fixes_to_numpy(f2, c2, 2)[0].tobytes() == fx.tobytes()
    assert (fx[:, 1]["status"] == abi.FIX_RECOVERED).sum() > 0
    _no_wrong_recovery(fx, cap["truth"]["epc"])


@pytest.mark.gpu
@pytest.mark.parametrize("P,W,snr_db", [(1, 1, 7.0), (32, 3, 7.0), (3, 3, 7.0), (12, 4, 0.0), (12, 4, 30.0)],
                         ids=["P1", "P32-W3", "W=P", "low-gate", "high-gate"])
def test_device_parameter_corners(rx, P, W, snr_db):
    from gen2_uhf_rfid_reader_b200 import capi
    cap = synth.make_capture(256, device="cpu", tag_gain=0.003, **WEAK)
    params = capi.default_recover_params(positions=P, max_flips=W, min_snr_db=snr_db)
    fx = _same_as_model(_device(rx, *_cuda(cap["iq"].numpy(), cap["segments"]), 2, params=params), params=params)
    st = fx[:, 1]["status"]
    if snr_db >= 30.0:
        assert (st == abi.FIX_RECOVERED).sum() == 0
    else:
        assert (st == abi.FIX_RECOVERED).sum() > 0
    assert (fx[:, 1]["n_flips"][st == abi.FIX_RECOVERED] <= W).all()


@pytest.mark.gpu
def test_device_writes_only_stored_records(rx):
    """segments with more windows than max_windows, with none, and with fewer: nothing is written beyond the stored
    records"""
    from gen2_uhf_rfid_reader_b200 import capi
    cap = synth.make_capture(8, device="cpu", tag_gain=0.003, **WEAK)
    n = int(cap["segments"]["length"][0])
    x = cap["iq"].numpy()
    segs = abi.make_segments([0, 0, 1000, 5, n], [x.size, 8 * n // 2, 40, 0, 6000])
    params = capi.default_recover_params(min_snr_db=-100.0)
    dev = _device(rx, *_cuda(x, segs), 3, params=params, sentinel=True)
    counts, fx = dev[2], dev[4]
    assert counts[0] > 3 and counts[1] > 3 and counts[2] == counts[3] == 0 and counts[4] == 1
    raw = fx.view(np.uint8).reshape(5, 3, 32)
    assert (raw[2:4] == 0xAB).all() and (raw[4, 1:] == 0xAB).all()
    assert (raw[:2] != 0xAB).any(axis=2).all() and (raw[4, 0] != 0xAB).any()
    _same_as_model(dev, params=params)


@pytest.mark.gpu
@pytest.mark.parametrize("q,tags", [(2, 4), (4, 8)], ids=["q2-4tags", "q4-8tags"])
def test_closed_loop_simulator_against_truth(q, tags):
    """rfid_b200_sim_capture, closed loop, tag_gain 0.004: no RECOVERED EPC differs from the simulator's epc; the EPC
    windows of empty slots are all SKIPPED; the first slots equal the restatement bit for bit"""
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = _rx(fixed_q=q)
    cap = rxq.sim_capture(capi.default_sim(n_tags=tags, closed_loop=1, seed=700 + q, tag_gain=0.004), 2048)
    res, cnt, quality, fixes = rxq.decode_capture_recover(cap["iq"], cap["segs"], max_windows=2)
    recs, counts = capi.results_to_numpy(res, cnt, 2)
    qq, _ = capi.quality_to_numpy(quality, cnt, 2)
    fx, _ = capi.fixes_to_numpy(fixes, cnt, 2)
    truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
    assert (counts == 2).all()
    n_rec = _no_wrong_recovery(fx, truth["epc"])
    empty = truth["n_replies"] == 0
    st = fx[:, 1]["status"]
    print("closed loop Q=%d: %d EPC ok, %d recovered, %d failing attempted; empty-slot EPC SNR max %.2f dB, failing "
          "reply SNR min %.2f dB" % (q, (recs[:, 1]["crc_ok"] == 1).sum(), n_rec,
                                     ((st >= abi.FIX_RECOVERED) & (st <= abi.FIX_FAILED)).sum(),
                                     10 * np.log10(qq[empty, 1]["snr"].max()),
                                     10 * np.log10(qq[~empty & (recs[:, 1]["crc_ok"] != 1), 1]["snr"].min())))
    assert (st[empty] == abi.FIX_SKIPPED).all()
    k = 64
    dev = _device(rxq, cap["iq"][:k * cap["segment_len"]], cap["segs"][:k], 2)
    assert _same_as_model(dev).tobytes() == fx[:k].tobytes()


@pytest.mark.gpu
def test_recover_epc_argument_checks(rx):
    """a NULL pointer (the quality buffer too), negative counts, P outside 1..32, W outside 1..P, a non-finite
    min_snr_db, more than 65536 candidates: RFID_B200_EINVAL, and nothing written"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    tap = torch.zeros(2 * rx.len_epc, dtype=torch.complex64, device="cuda")
    res = torch.zeros((2, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    qual = torch.zeros((2, 16), dtype=torch.uint8, device="cuda")
    out = torch.zeros((2, 32), dtype=torch.uint8, device="cuda")

    def call(w=tap.data_ptr(), r=res.data_ptr(), c=cnt.data_ptr(), q=qual.data_ptr(), o=out.data_ptr(), n=1, m=2,
             p=None):
        return L.rfid_b200_recover_epc(rx.h, w, r, c, q, n, m, p, o, None)

    assert call() == abi.OK and call(n=0) == abi.OK and call(m=0) == abi.OK
    for kw in (dict(w=None), dict(r=None), dict(c=None), dict(q=None), dict(o=None), dict(n=-1), dict(m=-1)):
        assert call(**kw) == abi.EINVAL, kw
    good = [dict(positions=1, max_flips=1), dict(positions=32, max_flips=4), dict(positions=16, max_flips=16)]
    bad = [dict(positions=0), dict(positions=33, max_flips=1), dict(max_flips=0), dict(positions=4, max_flips=5),
           dict(positions=32, max_flips=5), dict(positions=20, max_flips=20), dict(min_snr_db=float("nan")),
           dict(min_snr_db=float("inf")), dict(min_snr_db=float("-inf"))]
    for kw in good:
        assert call(p=C.byref(capi.default_recover_params(**kw))) == abi.OK, kw
    for kw in bad:
        assert call(p=C.byref(capi.default_recover_params(**kw))) == abi.EINVAL, kw
    with pytest.raises(capi.RfidB200Error):
        rx.recover_epc(tap, res, cnt, qual, 2, params=capi.default_recover_params(positions=0))
    torch.cuda.synchronize()
    assert (out == 0).all()
