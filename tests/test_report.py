"""Capture mode: the tag inventory report (rfid_b200_tag_report).

CPU: the numpy restatement (report_model.py) on hand-built record tables -- tags keyed by the full PC + EPC where the
READER_STATS key by one byte, rejections, slots that are not reads or not stored, counts out of range, power ties and
NaN, capacity -- and on the reference recording's records.  GPU: the device report equals the restatement bit for bit
on the hand-built tables, the recording (whole and segmented), the closed-loop simulator, a weak tag with recovered
reads, sc16 captures and adversarial 320,000-slot tables; the simulator's reports agree with its truth.
"""
import ctypes as C

import numpy as np
import pytest

import report_model as rpm
from gen2_uhf_rfid_reader_b200 import abi, synth


# ------------------------------------------------------------------ hand-built tables
def frame(payload, pc=0x30):
    """PC byte `pc` (0x30: 6 words) + 0x00 + 12-byte EPC + its CRC-16 -> uint8[16]"""
    b = bytes([pc, 0x00]) + bytes(bytearray(np.asarray(payload, dtype=np.uint8)))
    return np.frombuffer(b + synth.crc16_gen2(b).to_bytes(2, "big"), dtype=np.uint8).copy()


def table(nseg, mw):
    segs = abi.make_segments(np.arange(nseg, dtype=np.uint64) * 17000 + 5, np.full(nseg, 17000))
    recs = np.zeros((nseg, mw), dtype=abi.RESULT_DTYPE)
    recs["segment"] = np.arange(nseg)[:, None]
    recs["window"] = np.arange(mw)[None, :]
    recs["kind"] = np.arange(mw)[None, :] % 2            # RN16, EPC, RN16, ...
    recs["crc_ok"] = np.where(recs["kind"] == abi.EPC, 0, -1)
    recs["open_index"] = 300 + 900 * np.arange(mw)[None, :]
    recs["sync_index"] = 7
    recs["h_re"], recs["h_im"] = 0.5, -0.25
    return segs, recs, np.full(nseg, mw, dtype=np.int32)


def put(recs, s, k, bits, ok=1, h=None):
    recs[s, k]["kind"] = abi.EPC
    recs[s, k]["crc_ok"] = ok
    recs[s, k]["bits"] = bits
    recs[s, k]["tag_id"] = bits[13]
    if h is not None:
        recs[s, k]["h_re"], recs[s, k]["h_im"] = h


A = frame(np.arange(12) + 1)
B = A.copy()
B[2] ^= 0x80     # differs from A in bytes 2 and the CRC, not in byte 13
B = frame(B[2:14])
ONE_BIT = frame(np.bitwise_xor(A[2:14], np.eye(1, 12, 5, dtype=np.uint8)[0]))
LONG = frame(np.arange(12) + 1, pc=0x38)   # a 7-word length field


def case_byte13():
    segs, recs, counts = table(6, 2)
    for s, f in enumerate([A, B, A, B, B, A]):
        put(recs, s, 1, f)
    return dict(segs=segs, recs=recs, counts=counts)


def case_one_bit():
    segs, recs, counts = table(4, 2)
    for s, f in enumerate([A, ONE_BIT, ONE_BIT, A]):
        put(recs, s, 1, f)
    return dict(segs=segs, recs=recs, counts=counts)


def case_rejections():
    segs, recs, counts = table(6, 2)
    for s, f in enumerate([A, LONG, A, A, B, LONG]):
        put(recs, s, 1, f)
    q = np.zeros((6, 2), dtype=abi.QUALITY_DTYPE)
    q["outcome"] = abi.SLOT_SINGLE
    q["outcome"][2, 1] = q["outcome"][5, 1] = abi.SLOT_EMPTY   # slot 5: LONG and EMPTY: counted as a length rejection
    fx = np.zeros((6, 2), dtype=abi.EPC_FIX_DTYPE)
    fx["status"] = abi.FIX_NOT_EPC
    fx["status"][:, 1] = abi.FIX_CRC_OK
    recs[3, 1]["crc_ok"] = 0
    fx["status"][3, 1], fx["bits"][3, 1] = abi.FIX_RECOVERED, B            # a recovered read of B
    fx["status"][0, 0], fx["bits"][0, 0] = abi.FIX_RECOVERED, LONG         # a recovered read that fails the length test
    return dict(segs=segs, recs=recs, counts=counts, quality=q, fixes=fx)


def case_not_candidates():
    segs, recs, counts = table(5, 3)
    put(recs, 0, 1, A)
    put(recs, 1, 1, B, ok=0)                 # CRC failure
    recs[2, 0]["bits"] = A                   # an RN16 record holding EPC bytes
    recs[2, 0]["crc_ok"] = 1
    put(recs, 3, 2, B)                       # not stored: count 2
    counts[3] = 2
    put(recs, 4, 0, A)
    counts[4] = 0                            # nothing stored
    fx = np.zeros((5, 3), dtype=abi.EPC_FIX_DTYPE)
    fx["status"] = abi.FIX_FAILED
    fx["status"][3, 2], fx["bits"][3, 2] = abi.FIX_RECOVERED, A   # not stored either
    return dict(segs=segs, recs=recs, counts=counts, fixes=fx)


def case_counts():
    segs, recs, counts = table(5, 2)
    for s in range(5):
        put(recs, s, 0, A)
        put(recs, s, 1, B)
    counts[:] = [-5, 3, 1, 2, -1]
    return dict(segs=segs, recs=recs, counts=counts)


def case_power():
    """ties (also with +-0.0 components, which square to the same p) go to the lowest slot; NaN p ranks lowest"""
    segs, recs, counts = table(8, 2)
    nan = np.float32(np.nan)
    hs = [(0.5, 0.0), (-0.5, -0.0), (0.0, 0.5), (nan, 1.0), (0.25, 0.25), (-0.0, -0.5), (0.1, nan), (0.5, -0.0)]
    for s, h in enumerate(hs):
        put(recs, s, 1, A, h=h)
    put(recs, 3, 0, B, h=(nan, 0.0))         # B: only NaN powers
    put(recs, 6, 0, B, h=(0.0, nan))
    put(recs, 7, 0, LONG, h=(9.0, 9.0))
    return dict(segs=segs, recs=recs, counts=counts, check_length=0)


def case_capacity():
    segs, recs, counts = table(40, 2)
    rng = np.random.default_rng(3)
    pool = [frame(rng.integers(0, 256, 12)) for _ in range(12)]
    for s in range(40):
        put(recs, s, 1, pool[rng.integers(0, 12)])
        if s % 3 == 0:
            put(recs, s, 0, pool[rng.integers(0, 12)])
    return dict(segs=segs, recs=recs, counts=counts, max_tags=5)


def case_random(seed, nseg=300, mw=3):
    """every field drawn: kinds, CRC flags, counts in [-2, mw + 2], a pool of keys with near neighbours, quality and
    fixes, powers with zeros, NaN and ties, times with large offsets"""
    rng = np.random.default_rng(seed)
    segs, recs, counts = table(nseg, mw)
    segs["offset"] = rng.integers(0, 1 << 40, nseg).astype(np.uint64)
    pool = [frame(rng.integers(0, 256, 12)) for _ in range(20)]
    pool += [p.copy() for p in pool[:5]]
    for p in pool[-5:]:
        p[rng.integers(0, 16)] ^= np.uint8(1 << rng.integers(0, 8))
    pool.append(LONG)
    flat = recs.reshape(-1)
    n = flat.size
    flat["kind"] = rng.integers(0, 2, n)
    flat["crc_ok"] = np.where(flat["kind"] == abi.EPC, rng.integers(0, 2, n), -1)
    flat["bits"] = np.array(pool)[rng.integers(0, len(pool), n)]
    flat["open_index"] = rng.integers(-100, 1 << 20, n)
    flat["sync_index"] = rng.integers(-3, 40, n)
    h = rng.choice(np.array([0.0, -0.0, 0.5, -0.5, 0.25, np.nan, 1e-3], dtype=np.float32), size=(n, 2))
    drawn = rng.random((n, 2)) < 0.5
    h[drawn] = rng.standard_normal(int(drawn.sum())).astype(np.float32)
    flat["h_re"], flat["h_im"] = h[:, 0], h[:, 1]
    counts[:] = rng.integers(-2, mw + 3, nseg)
    q = np.zeros((nseg, mw), dtype=abi.QUALITY_DTYPE)
    q["outcome"] = rng.integers(0, 3, (nseg, mw))
    fx = np.zeros((nseg, mw), dtype=abi.EPC_FIX_DTYPE)
    fx["status"] = rng.integers(0, 6, (nseg, mw))
    fx["bits"] = np.array(pool)[rng.integers(0, len(pool), (nseg, mw))]
    return dict(segs=segs, recs=recs, counts=counts, quality=q, fixes=fx, max_tags=int(rng.integers(0, 30)),
                check_length=int(rng.integers(0, 2)))


CASES = {"byte13": case_byte13, "one_bit": case_one_bit, "rejections": case_rejections,
         "not_candidates": case_not_candidates, "counts": case_counts, "power": case_power, "capacity": case_capacity,
         "random1": lambda: case_random(1), "random2": lambda: case_random(2, nseg=1500, mw=2)}


def model(c):
    return rpm.report(c["segs"], c["recs"], c["counts"], quality=c.get("quality"), fixes=c.get("fixes"),
                      check_length=c.get("check_length", 1), max_tags=c.get("max_tags", 1024))


# ------------------------------------------------------------------ CPU: the rule
def test_full_epc_against_the_one_byte_tag_id(oracle):
    """two EPCs that share bits 104..111 are two tags in the report and one tag_id in the READER_STATS replay"""
    c = case_byte13()
    assert A[13] == B[13] and (A != B).any()
    tags, sm, rt = model(c)
    assert sm["n_tags"] == 2 and tags["reads"].tolist() == [3, 3]
    assert [t.tobytes() for t in tags["epc"]] == [A.tobytes(), B.tobytes()]
    assert rt.reshape(6, 2)[:, 1].tolist() == [0, 1, 0, 1, 1, 0] and (rt.reshape(6, 2)[:, 0] == -1).all()
    st = oracle.reduce_stats(c["recs"], c["counts"], True)
    assert st.tag_map() == {int(A[13]): 6}


def test_one_bit_apart():
    tags, sm, rt = model(case_one_bit())
    assert sm["n_tags"] == 2 and tags["reads"].tolist() == [2, 2]
    assert tags["first_slot"].tolist() == [1, 3] and tags["last_slot"].tolist() == [7, 5]


def test_rejections():
    """the length field (records and fixes) and EMPTY slots: read_tag -2, counted once under the first test failed"""
    c = case_rejections()
    tags, sm, rt = model(c)
    rt = rt.reshape(6, 2)
    assert rt[:, 1].tolist() == [0, -2, -2, 1, 1, -2] and rt[0, 0] == -2 and (rt[1:, 0] == -1).all()
    assert (sm["reads"], sm["recovered"], sm["rejected_length"], sm["rejected_empty"]) == (3, 1, 3, 1)
    # B is the recovered read of segment 3 and the record of segment 4: one tag
    assert sm["n_tags"] == 2 and tags["reads"].tolist() == [1, 2] and tags["recovered"].tolist() == [0, 1]
    assert [e.tobytes() for e in tags["epc"]] == [A.tobytes(), B.tobytes()]
    tags0, sm0, _ = rpm.report(c["segs"], c["recs"], c["counts"], quality=c["quality"], fixes=c["fixes"],
                               check_length=0)
    assert sm0["rejected_length"] == 0 and sm0["rejected_empty"] == 2 and sm0["n_tags"] == 3


def test_not_candidates_and_not_stored():
    tags, sm, rt = model(case_not_candidates())
    rt = rt.reshape(5, 3)
    assert rt[0].tolist() == [-1, 0, -1] and rt[1].tolist() == [-1, -1, -1] and rt[2].tolist() == [-1, -1, -1]
    assert rt[3].tolist() == [-1, -1, rpm.NOT_STORED] and (rt[4] == rpm.NOT_STORED).all()
    assert sm["n_tags"] == 1 and sm["reads"] == 1


def test_counts_out_of_range():
    tags, sm, rt = model(case_counts())
    rt = rt.reshape(5, 2)
    assert (rt[0] == rpm.NOT_STORED).all() and (rt[4] == rpm.NOT_STORED).all()
    assert rt[1].tolist() == [0, 1] and rt[2].tolist() == [0, rpm.NOT_STORED] and rt[3].tolist() == [0, 1]
    assert tags["reads"].tolist() == [3, 2]


def test_power_ties_and_nan():
    tags, sm, rt = model(case_power())
    a, b, l = tags   # A first read at slot 1, B at slot 6, LONG at slot 14
    assert a["peak_slot"] == 1 and a["peak_power"] == np.float32(0.25)     # slots 1, 3, 5, 11, 15 tie; 7 is NaN
    assert b["peak_slot"] == 6 and b["peak_power"].view(np.uint32) == rpm.NAN_BITS and b["reads"] == 2
    assert l["peak_power"] == np.float32(162.0)
    assert a["last_slot"] == 15 and a["last_h_re"] == np.float32(0.5) and np.signbit(a["last_h_im"])


def test_capacity():
    c = case_capacity()
    tags, sm, rt = model(c)
    full, _, rt_full = rpm.report(c["segs"], c["recs"], c["counts"], max_tags=1024)
    assert sm["n_tags"] == full.size > 5 and tags.size == 5
    assert tags.tobytes() == full[:5].tobytes() and (rt == rt_full).all() and rt.max() == sm["n_tags"] - 1


def test_times():
    """first_time / last_time = offset + decim * (open_index + sync_index) in raw samples"""
    c = case_one_bit()
    tags, _, _ = model(c)
    r = c["recs"]
    assert tags["first_time"][0] == int(c["segs"]["offset"][0]) + 5 * (int(r[0, 1]["open_index"]) + 7)
    assert tags["last_time"][0] == int(c["segs"]["offset"][3]) + 5 * (int(r[3, 1]["open_index"]) + 7)


def test_recording(cfg1_golden, oracle):
    """the reference's records of its recording: one tag, 70 reads, byte 13 = 0x27 (README: 70 EPCs correct, tag
    0x27), as the READER_STATS replay counts it"""
    recs = cfg1_golden[None, :]
    segs = abi.make_segments([0], [1247958])
    tags, sm, rt = rpm.report(segs, recs, np.array([recs.shape[1]]))
    assert sm["n_tags"] == 1 and tags[0]["reads"] == 70 and tags[0]["epc"][13] == 0x27 and sm["recovered"] == 0
    assert sm["rejected_length"] == 0 and (tags[0]["epc"][0] >> 3) == 6
    assert oracle.reduce_stats(recs, np.array([recs.shape[1]]), True).tag_map() == {0x27: 70}


def test_tag_table():
    from gen2_uhf_rfid_reader_b200 import capi
    tags, _, _ = model(case_one_bit())
    t = capi.tag_table(tags, ntaps=25, adc_rate=2_000_000)
    assert t["epc"][0] == A.tobytes().hex() and t["reads"].tolist() == [2, 2]
    assert t["first_us"][0] == tags["first_time"][0] / 2.0
    assert abs(t["peak_rssi_db"][0] - 10 * np.log10((0.5 ** 2 + 0.25 ** 2) / 625)) < 1e-5
    assert abs(t["last_phase_deg"][0] - np.degrees(np.arctan2(-0.25, 0.5))) < 1e-9


def test_defaults_layouts_and_null_context():
    from gen2_uhf_rfid_reader_b200 import capi
    rp = capi.default_report_params()
    assert rp.check_length == 1 and list(rp.reserved) == [0] * 7
    assert C.sizeof(abi.ReportParams) == 32 and C.sizeof(abi.Tag) == 64 and C.sizeof(abi.TagSummary) == 32
    assert abi.TAG_DTYPE == rpm.TAG_DTYPE and abi.TAG_SUMMARY_DTYPE == rpm.TAG_SUMMARY_DTYPE
    for st, dt in ((abi.Tag, abi.TAG_DTYPE), (abi.TagSummary, abi.TAG_SUMMARY_DTYPE)):
        for name, _ in st._fields_:
            assert getattr(st, name).offset == dt.fields[name][1], name
    assert "rfid_b200_tag_report" in capi.EXPORTED_SYMBOLS and "rfid_b200_default_report_params" in capi.EXPORTED_SYMBOLS
    L = capi.load_library()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    assert L.rfid_b200_tag_report(None, p, p, p, 1, 1, None, None, None, 1, p, p, None, None) == abi.EINVAL
    L.rfid_b200_default_report_params(None)   # tolerated


# ------------------------------------------------------------------ GPU
def _rx(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx(**kw)


@pytest.fixture(scope="module")
def rx():
    return _rx()


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def _device(rx, c, sentinel=-7):
    """the hand-built case c on the device: (tags, summary, read_tag) as host numpy, read_tag prefilled with sentinel"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    recs = c["recs"]
    nseg, mw = recs.shape
    res, cnt = _t(recs), torch.from_numpy(np.asarray(c["counts"], dtype=np.int32)).cuda()
    q = _t(c["quality"]) if c.get("quality") is not None else None
    f = _t(c["fixes"]) if c.get("fixes") is not None else None
    rt = torch.full((nseg * mw,), sentinel, dtype=torch.int32, device="cuda")
    params = capi.default_report_params(check_length=c.get("check_length", 1))
    tags, summary, rt = rx.tag_report(res, cnt, capi.segments_to_device(c["segs"], "cuda"), mw, quality=q, fixes=f,
                                      params=params, max_tags=c.get("max_tags", 1024), read_tag=rt)
    torch.cuda.synchronize()
    t, sm = capi.tags_to_numpy(tags, summary)
    return t, sm, rt.cpu().numpy()


def _same_as_model(dev, want, sentinel=-7):
    t, sm, rt = dev
    wt, wsm, wrt = want
    assert sm.tobytes() == wsm.tobytes(), (sm, wsm)
    assert t.tobytes() == wt.tobytes()
    stored = wrt != rpm.NOT_STORED
    assert (rt[stored] == wrt[stored]).all() and (rt[~stored] == sentinel).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_hand_built(rx, name):
    c = CASES[name]()
    _same_as_model(_device(rx, c), model(c))
    assert rx.last_launch_count() == 5


def _report_of(rx, out, segs_np, max_windows, max_tags=1024):
    """decode_capture_report output -> host (recs, counts, quality, fixes, model report, device report)"""
    from gen2_uhf_rfid_reader_b200 import capi
    res, cnt, qual, fix, tags, summary, rt = out
    recs, counts = capi.results_to_numpy(res, cnt, max_windows)
    q = capi.quality_to_numpy(qual, cnt, max_windows)[0] if qual is not None else None
    fx = capi.fixes_to_numpy(fix, cnt, max_windows)[0] if fix is not None else None
    want = rpm.report(segs_np, recs, counts, quality=q, fixes=fx, max_tags=max_tags, decim=rx.params.decim)
    t, sm = capi.tags_to_numpy(tags, summary)
    dev = (t, sm, rt.cpu().numpy())
    _same_as_model(dev, want, sentinel=-1)
    return recs, counts, q, fx, dev


@pytest.mark.gpu
def test_device_on_the_recording(rx, cfg1_iq):
    """the recording decoded whole and as its 72 ingest segments: equal to the restatement; the two reports agree in
    EPC, reads, first and last time, and in peak power within the score drift of segmenting"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    iq = torch.from_numpy(cfg1_iq.copy()).cuda()
    whole = abi.make_segments([0], [cfg1_iq.size])
    _, _, _, _, (t1, s1, _) = _report_of(rx, rx.decode_capture_report(iq, capi.segments_to_device(whole, "cuda"), 160),
                                         whole, 160)
    segs, _, _ = rx.ingest_capture_host(cfg1_iq, max_windows=4)
    assert segs.size == 72
    _, _, _, _, (t2, s2, _) = _report_of(rx, rx.decode_capture_report(iq, capi.segments_to_device(segs, "cuda"), 4),
                                         segs, 4)
    assert s1["n_tags"] == s2["n_tags"] == 1 and t1[0]["reads"] == t2[0]["reads"] == 70 and t1[0]["epc"][13] == 0x27
    for f in ("epc", "reads", "recovered", "first_time", "last_time"):
        assert t1[f].tobytes() == t2[f].tobytes(), f
    assert abs(t1[0]["peak_power"] / t2[0]["peak_power"] - 1) < 1e-3
    print("recording: %s" % capi.tag_table(t1))


@pytest.mark.gpu
@pytest.mark.parametrize("q,tags", [(2, 4), (4, 8)], ids=["q2-4tags", "q4-8tags"])
def test_closed_loop_simulator_against_truth(q, tags):
    """the reported EPCs are the truth EPCs with at least one passing EPC window; per EPC, reads = the slots whose
    replier sent it and whose window passed; no other tag"""
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = _rx(fixed_q=q)
    cap = rxq.sim_capture(capi.default_sim(n_tags=tags, closed_loop=1, seed=900 + q), 2048)
    segs = cap["segs"].cpu().numpy().view(abi.SEGMENT_DTYPE).reshape(-1)
    recs, counts, qq, fx, (t, sm, rt) = _report_of(rxq, rxq.decode_capture_report(cap["iq"], cap["segs"], 2), segs, 2)
    truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
    assert (counts == 2).all()
    passed = rt.reshape(-1, 2)[:, 1] >= 0
    assert (truth["replier"][passed] >= 0).all()
    want = {}
    for s in np.nonzero(passed)[0]:
        want[truth["epc"][s].tobytes()] = want.get(truth["epc"][s].tobytes(), 0) + 1
    got = {e.tobytes(): int(n) for e, n in zip(t["epc"], t["reads"])}
    assert got == want and len(got) == sm["n_tags"] > 1
    for s in np.nonzero(passed)[0]:
        assert t[rt[2 * s + 1]]["epc"].tobytes() == truth["epc"][s].tobytes()
    print("closed loop Q=%d: %d tags, %d reads, %d rejected as empty" % (q, sm["n_tags"], sm["reads"],
                                                                         sm["rejected_empty"]))


@pytest.mark.gpu
def test_weak_tag_with_fixes(rx):
    """make_capture(600, seed=77, tag_gain=0.003): reads = CRC-passing + recovered, recovered = the RECOVERED fixes"""
    from gen2_uhf_rfid_reader_b200 import capi
    cap = synth.make_capture(600, device="cpu", seed=77, tag_gain=0.003)
    iq = cap["iq"].cuda()
    recs, counts, q, fx, (t, sm, _) = _report_of(rx, rx.decode_capture_report(iq, capi.segments_to_device(
        cap["segments"], "cuda"), 2), cap["segments"], 2)
    n_ok = int((recs[:, 1]["crc_ok"] == 1).sum())
    n_rec = int((fx["status"] == abi.FIX_RECOVERED).sum())
    assert (n_ok, n_rec) == (388, 114) and sm["n_tags"] == 1
    assert t[0]["epc"].tobytes() == cap["truth"]["epc"][0].tobytes()
    # a reply this weak mostly measures below the quality rule's empty_db: those reads are rejected as EMPTY
    print("weak tag: %d reads, %d recovered, %d rejected as empty" % (sm["reads"], sm["recovered"], sm["rejected_empty"]))
    assert sm["reads"] + sm["rejected_empty"] == n_ok + n_rec and sm["rejected_length"] == 0
    # without the EMPTY rejection every CRC-passing and every recovered read counts
    out = rx.decode_capture_report(iq, capi.segments_to_device(cap["segments"], "cuda"), 2, reject_empty=False)
    assert out[2] is not None
    _, _, _, _, (t1, sm1, _) = _report_of(rx, out[:2] + (None,) + out[3:], cap["segments"], 2)
    assert t1[0]["reads"] == sm1["reads"] == n_ok + n_rec and t1[0]["recovered"] == sm1["recovered"] == n_rec
    out = rx.decode_capture_report(iq, capi.segments_to_device(cap["segments"], "cuda"), 2, recover=False,
                                   reject_empty=False)
    assert out[3] is None
    _, _, _, _, (t0, sm0, _) = _report_of(rx, out[:2] + (None,) + out[3:], cap["segments"], 2)
    assert t0[0]["reads"] == n_ok and sm0["recovered"] == 0


@pytest.mark.gpu
def test_sc16_equals_fc32_and_calls_repeat(rx):
    """an sc16 capture and its fc32 conversion give identical reports; a second call gives the same bytes"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    from test_sc16 import SCALES, convert, quantise
    cap = synth.make_capture(256, device="cpu", seed=78, fixed_q=4, n_tags=8, tag_gain=0.004)
    q16 = quantise(cap["iq"].numpy(), SCALES[0])
    segs = capi.segments_to_device(cap["segments"], "cuda")
    a = rx.decode_capture_report(torch.from_numpy(q16).cuda(), segs, 2, scale=SCALES[0])
    b = rx.decode_capture_report(torch.from_numpy(convert(q16, SCALES[0]).copy()).cuda(), segs, 2)
    c = rx.decode_capture_report(torch.from_numpy(convert(q16, SCALES[0]).copy()).cuda(), segs, 2)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(y, z)
    _report_of(rx, a, cap["segments"], 2)


def _big(distinct, nseg=160000, seed=11):
    """nseg x 2 slots, every one an EPC read (crc_ok 1; the report trusts the flag): of one EPC, or all distinct"""
    rng = np.random.default_rng(seed)
    segs, recs, counts = table(nseg, 2)
    flat = recs.reshape(-1)
    flat["kind"], flat["crc_ok"] = abi.EPC, 1
    if distinct:
        bits = np.zeros((flat.size, 16), dtype=np.uint8)
        bits[:, 0] = 0x30
        bits[:, 2:10] = rng.permutation(flat.size).astype(">u8").view(np.uint8).reshape(-1, 8)
        bits[:, 10:16] = rng.integers(0, 256, (flat.size, 6))
        flat["bits"] = bits
    else:
        flat["bits"] = A
    flat["h_re"] = rng.choice(np.array([0.5, -0.5, 0.25, np.nan], dtype=np.float32), flat.size)
    flat["h_im"] = rng.choice(np.array([0.0, -0.0, 0.25], dtype=np.float32), flat.size)
    return dict(segs=segs, recs=recs, counts=counts)


@pytest.mark.gpu
@pytest.mark.parametrize("distinct,max_tags", [(False, 1024), (True, 400000), (True, 1000)],
                         ids=["one-epc", "distinct", "distinct-over-capacity"])
def test_device_adversarial(rx, distinct, max_tags):
    c = _big(distinct)
    c["max_tags"] = max_tags
    dev = _device(rx, c)
    want = model(c)
    _same_as_model(dev, want)
    assert dev[1]["n_tags"] == (320000 if distinct else 1) and dev[1]["reads"] == 320000


@pytest.mark.gpu
def test_tag_report_argument_checks(rx):
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    segs = torch.zeros((2, 16), dtype=torch.uint8, device="cuda")
    res = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    tags = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    sm = torch.zeros(32, dtype=torch.uint8, device="cuda")

    def call(h=rx.h, s=segs.data_ptr(), r=res.data_ptr(), c=cnt.data_ptr(), n=2, m=2, p=None, mt=4,
             t=tags.data_ptr(), o=sm.data_ptr()):
        return L.rfid_b200_tag_report(h, s, r, c, n, m, None, None, p, mt, t, o, None, None)

    assert call() == abi.OK and call(n=0) == abi.OK and call(m=0) == abi.OK and call(mt=0, t=None) == abi.OK
    for kw in (dict(h=None), dict(s=None), dict(r=None), dict(c=None), dict(o=None), dict(t=None), dict(n=-1),
               dict(m=-1), dict(mt=-1), dict(n=1 << 16, m=1 << 15), dict(n=(1 << 30) + 1, m=2)):
        assert call(**kw) == abi.EINVAL, kw
    for v in (-1, 2):
        assert call(p=C.byref(capi.default_report_params(check_length=v))) == abi.EINVAL
    assert call(p=C.byref(capi.default_report_params(check_length=0))) == abi.OK
    torch.cuda.synchronize()
    assert (tags == 0).all()
