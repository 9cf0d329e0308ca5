"""Capture mode: attribution of failing EPC replies to a dictionary of known frames (rfid_b200_match_epc).

CPU: the numpy restatement (match_model.py) on hand-built windows -- exact signs, ties, duplicates, K = 1 and 0, the
reliability cap, S1 = 0, status precedence, the live count -- the int8 product form against the direct cost, and the
reference recording.  GPU: the device records and per-entry counts equal the restatement bit for bit on the hand-built
windows, the recording (whole and as its 72 ingest segments), weak simulated tags (fc32 and sc16) and a large
adversarial dictionary; against the simulator's truth no MATCHED window names the wrong tag, and matching reads more
replies than recovery does.
"""
import ctypes as C

import numpy as np
import pytest

import match_model as mm
import quality_model as qm
import recover_model as rm
from gen2_uhf_rfid_reader_b200 import abi, synth

N_I, N_F, _, LEN_EPC = qm.derived(2_000_000)
SYNC, T = 20, np.float32(N_F / 2)


def signs_to_frame(s):
    """codeword signs [128] -> the frame whose FM0 signs they are"""
    s = np.asarray(s, dtype=bool)
    return np.packbits((s ^ np.concatenate([[True], s[:-1]])).astype(np.uint8))


def random_signs(rng, n=1):
    return rng.integers(0, 2, size=(n, 128)).astype(bool)


def hand_window(r):
    """a window tap row and EPC record whose projections are exactly r (float32 [128], values exact when halved)"""
    a, b, _, _ = qm.positions(1, SYNC, T, N_F, 0)
    assert np.unique(np.concatenate([a, b])).size == 256 and b.max() < LEN_EPC
    w = np.zeros(LEN_EPC, dtype=np.complex64)
    w[a] = np.float32(r) / 2
    w[b] = -np.float32(r) / 2
    rec = np.zeros((), dtype=abi.RESULT_DTYPE)
    rec["kind"], rec["crc_ok"], rec["sync_index"], rec["T"] = abi.EPC, 0, SYNC, T
    rec["h_re"], rec["length"] = 1.0, LEN_EPC
    return w, rec


def table(rows):
    """rows: list of (r or None, kind, crc_ok) -> windows [1, n, L], recs [1, n], counts [1]"""
    n = len(rows)
    wins = np.zeros((1, n, LEN_EPC), dtype=np.complex64)
    recs = np.zeros((1, n), dtype=abi.RESULT_DTYPE)
    for k, (r, kind, ok) in enumerate(rows):
        w, rec = hand_window(np.zeros(128, np.float32) if r is None else r)
        rec["kind"], rec["crc_ok"], rec["window"] = kind, ok, k
        wins[0, k], recs[0, k] = w, rec
    return wins, recs, np.array([n], dtype=np.int32)


def proj(signs, mag=1.0):
    return np.where(signs, np.float32(1), np.float32(-1)) * np.asarray(mag, dtype=np.float32)


def hand_cases():
    """named (windows, recs, counts, dictionary, fixes, n_dict, expectations) of the hand-built windows"""
    rng = np.random.default_rng(7)
    S = random_signs(rng, 6)
    F = np.array([signs_to_frame(s) for s in S])
    cases = {}
    # exact signs: cost 0 against its own entry
    w, r, c = table([(proj(S[0]), 1, 0)])
    cases["exact"] = (w, r, c, F[:4], None, None, dict(entry=0, cost=0, status=mm.MATCHED))
    # ties: entries one sign from the window at different positions, equal q, cost 16 each -> the lower index
    s1, s2 = S[0].copy(), S[0].copy()
    s1[10] ^= True
    s2[90] ^= True
    w, r, c = table([(proj(S[0]), 1, 0)])
    cases["tie"] = (w, r, c, np.array([F[1], signs_to_frame(s2), signs_to_frame(s1)]), None, None,
                    dict(entry=1, cost=16, runner_up=16, status=mm.AMBIGUOUS))
    # duplicate entries: D2 = D1, AMBIGUOUS
    cases["duplicate"] = (w, r, c, np.array([F[2], F[0], F[0]]), None, None,
                          dict(entry=1, cost=0, runner_up=0, status=mm.AMBIGUOUS))
    # K = 1: runner_up INT32_MAX
    cases["k1"] = (w, r, c, F[:1], None, None, dict(entry=0, cost=0, runner_up=mm.INT32_MAX, status=mm.MATCHED))
    # K = 0 (a dictionary of max_dict 2 with n_dict 0)
    cases["k0"] = (w, r, c, F[:2], None, 0, dict(entry=-1, cost=mm.INT32_MAX, runner_up=mm.INT32_MAX,
                                                 status=mm.NO_MATCH, n_diff=-1))
    # the q cap: one sign 1000x the others is wrong; it costs 127, not rint(16 * 1000 / mean) = 1817
    mag = np.ones(128, np.float32)
    mag[5] = 1000.0
    sw = S[0].copy()
    sw[5] ^= True
    w, r, c = table([(proj(sw, mag), 1, 0)])
    cases["cap"] = (w, r, c, F[:1], None, None, dict(entry=0, cost=127, n_diff=1, status=mm.MATCHED))
    # S1 = 0: SKIPPED
    w, r, c = table([(None, 1, 0)])
    cases["s1_zero"] = (w, r, c, F[:3], None, None, dict(entry=-1, cost=-1, status=mm.SKIPPED))
    # precedence: RN16, EPC passing, EPC failing with a RECOVERED fix, EPC with no decisions, attempted
    rows = [(proj(S[0]), 0, -1), (proj(S[0]), 1, 1), (proj(S[0]), 1, 0), (proj(S[0]), 1, -2), (proj(S[3]), 1, 0)]
    w, r, c = table(rows)
    fx = np.zeros((1, 5), dtype=abi.EPC_FIX_DTYPE)
    fx["status"] = [abi.FIX_NOT_EPC, abi.FIX_CRC_OK, abi.FIX_RECOVERED, abi.FIX_SKIPPED, abi.FIX_FAILED]
    want_fix = [mm.NOT_EPC, mm.ALREADY_READ, mm.ALREADY_READ, mm.SKIPPED, mm.MATCHED]
    want_nofix = [mm.NOT_EPC, mm.ALREADY_READ, mm.MATCHED, mm.SKIPPED, mm.MATCHED]
    cases["precedence_fixes"] = (w, r, c, F[:4], fx, None, dict(statuses=want_fix))
    cases["precedence"] = (w, r, c, F[:4], None, None, dict(statuses=want_nofix))
    # n_dict below and above max_dict: 1 of 4 entries live (the window's own entry, 3, is not), 9 clamps to 4
    w, r, c = table([(proj(S[3]), 1, 0)])
    cases["n_dict_below"] = (w, r, c, F[:4], None, 1, dict(entry=0, status=mm.NO_MATCH))
    cases["n_dict_above"] = (w, r, c, F[:4], None, 9, dict(entry=3, cost=0, status=mm.MATCHED))
    return cases


def _check(out, cnt, exp, dictionary):
    if "statuses" in exp:
        assert out[0]["status"].tolist() == exp["statuses"]
    else:
        for k, v in exp.items():
            assert int(out[0, 0][k]) == v, (k, out[0, 0])
    m = (out["status"] == mm.MATCHED).reshape(-1)
    assert cnt.size == len(dictionary) and int(cnt["matched"].sum()) == int(m.sum())


# ------------------------------------------------------------------ CPU: the rule
@pytest.mark.parametrize("name", list(hand_cases()))
def test_hand_built(name):
    w, r, c, d, fx, nd, exp = hand_cases()[name]
    out, cnt = mm.match(w, r, c, d, fixes=fx, n_dict=nd)
    _check(out, cnt, exp, d)


def test_reliabilities():
    """q_j = min(127, rint(16 |r_j| / mean |r|)), ties to even; S1 = 0 and NaN are not ok"""
    r = np.ones((3, 128), np.float32)
    r[0, 0] = 1000.0
    r[1, :] = 0.0
    r[2, 3] = np.nan
    q, s, ok = mm.reliabilities(r)
    assert ok.tolist() == [True, False, False] and q[0, 0] == 127
    m = (1000.0 + 127) / 128
    assert q[0, 1] == np.rint(16 / m)
    r = np.full((1, 128), 2.0, np.float32)
    r[0, :2] = [1.0, 3.0]    # mean 2: 8 and 24 exactly; a half step rounds to even
    r[0, 2:4] = [2.0 + 1 / 16, 2.0 - 1 / 16]
    q, _, _ = mm.reliabilities(r)
    assert q[0, :4].tolist() == [8, 24, 16, 16]


def test_product_form_equals_the_direct_cost():
    rng = np.random.default_rng(3)
    q = rng.integers(0, 128, size=(50, 128))
    s = random_signs(rng, 50)
    cw = random_signs(rng, 300).astype(np.uint8)
    assert (mm.costs(q, s, cw) == mm.costs_gemm(q, s, cw)).all()
    assert (mm.costs(q[:1], s[:1], s[:1].astype(np.uint8)) == 0).all()
    f = rng.integers(0, 256, size=(20, 16)).astype(np.uint8)
    for fr, cs in zip(f, mm.codeword_signs(f)):   # the signs are recover_model's FM0 rule
        r = np.where(cs, 1.0, -1.0).astype(np.float32)
        assert rm.sign_errors(r, fr).size == 0


@pytest.fixture(scope="module")
def rec_windows(oracle, cfg1_iq):
    return qm.oracle_windows(oracle, cfg1_iq, abi.make_segments([0], [cfg1_iq.size]), 160)


def test_recording(rec_windows):
    """the tag's frame as the dictionary: 71 NOT_EPC, 70 ALREADY_READ; the failing EPC window, whose tag no longer
    answered (its decision SNR is that of noise), is NO_MATCH"""
    w, r, c = rec_windows
    n = int(c[0])
    ok = np.nonzero((r[0, :n]["kind"] == abi.EPC) & (r[0, :n]["crc_ok"] == 1))[0]
    d = r[0, ok[0]]["bits"][None].copy()
    out, cnt = mm.match(w, r, c, d)
    st = out[0, :n]["status"]
    assert (st == mm.NOT_EPC).sum() == 71 and (st == mm.ALREADY_READ).sum() == 70 and (st == mm.NO_MATCH).sum() == 1
    bad = out[0, np.nonzero(st == mm.NO_MATCH)[0][0]]
    print("recording: failing EPC window costs %.2f mean reliabilities (n_diff %d)" % (bad["cost"] / 16, bad["n_diff"]))
    assert bad["cost"] > 16 * mm.DEFAULT_MAX_COST and cnt["matched"].tolist() == [0]


def test_defaults_layouts_and_null_context():
    from gen2_uhf_rfid_reader_b200 import capi
    mp = capi.default_match_params()
    assert (mp.max_cost, mp.min_margin) == (np.float32(mm.DEFAULT_MAX_COST), np.float32(mm.DEFAULT_MIN_MARGIN))
    assert list(mp.reserved) == [0] * 6
    assert abi.EPC_MATCH_DTYPE == mm.EPC_MATCH_DTYPE and abi.MATCH_COUNT_DTYPE == mm.MATCH_COUNT_DTYPE
    for st, dt in ((abi.EpcMatch, abi.EPC_MATCH_DTYPE), (abi.MatchCount, abi.MATCH_COUNT_DTYPE)):
        for name, _ in st._fields_:
            assert getattr(st, name).offset == dt.fields[name][1]
    assert (abi.MATCH_ALREADY_READ, abi.MATCH_MATCHED, abi.MATCH_AMBIGUOUS, abi.MATCH_NO_MATCH, abi.MATCH_SKIPPED,
            abi.MATCH_NOT_EPC) == (mm.ALREADY_READ, mm.MATCHED, mm.AMBIGUOUS, mm.NO_MATCH, mm.SKIPPED, mm.NOT_EPC)
    assert "rfid_b200_match_epc" in capi.EXPORTED_SYMBOLS and "rfid_b200_default_match_params" in capi.EXPORTED_SYMBOLS
    L = capi.load_library()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    assert L.rfid_b200_match_epc(None, p, p, p, None, 1, 1, p, None, 1, None, p, None, None) == abi.EINVAL
    L.rfid_b200_default_match_params(None)   # tolerated


def test_tag_table_matched_column():
    """without matched= the table is what it was; with it, one more column after `recovered`"""
    from gen2_uhf_rfid_reader_b200 import capi
    t = np.zeros(2, dtype=abi.TAG_DTYPE)
    t["reads"], t["peak_power"], t["last_h_re"] = [3, 4], 625.0, 1.0
    plain = capi.tag_table(t)
    assert plain.dtype == capi.TAG_TABLE_DTYPE
    m = capi.tag_table(t, matched=np.array([5, 6, 7]))
    assert m.dtype.names == plain.dtype.names[:3] + ("matched",) + plain.dtype.names[3:]
    assert m["matched"].tolist() == [5, 6]
    for n in plain.dtype.names:
        assert m[n].tobytes() == plain[n].tobytes()


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rx():
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx()


def _upload(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _device_on(rx, w, r, c, d, fixes=None, n_dict=None, params=None):
    """match_epc on host-built windows / records: (EPC_MATCH_DTYPE [nseg, mw], MATCH_COUNT_DTYPE [max_dict]); the
    match buffer starts as 0xAB bytes so that a write to an unstored slot shows"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    nseg, mw = r.shape
    tap = _upload(w.reshape(-1))
    res = _upload(r.view(np.uint8).reshape(-1, 64))
    cnt = _upload(c.astype(np.int32))
    fx = _upload(fixes.view(np.uint8).reshape(-1, 32)) if fixes is not None else None
    nd = _upload(np.array([n_dict], np.int32)) if n_dict is not None else None
    match = torch.full((nseg * mw, 32), 0xAB, dtype=torch.uint8, device="cuda")
    match, mc = rx.match_epc(tap, res, cnt, np.asarray(d, np.uint8).reshape(-1, 16), mw, fixes=fx, n_dict=nd,
                             params=params, match=match)
    torch.cuda.synchronize()
    return capi.matches_to_numpy(match, cnt, mw, mc)


def _same_as_model(rx, w, r, c, d, fixes=None, n_dict=None, params=None):
    kw = dict(max_cost=params.max_cost, min_margin=params.min_margin) if params is not None else {}
    got, gc = _device_on(rx, w, r, c, d, fixes, n_dict, params)
    want, wc = mm.match(w, r, c, d, fixes=fixes, n_dict=n_dict, **kw)
    stored = np.arange(r.shape[1])[None, :] < np.minimum(np.maximum(c, 0), r.shape[1])[:, None]
    assert got[stored].tobytes() == want[stored].tobytes()
    assert (got.view(np.uint8).reshape(r.shape + (32,))[~stored] == 0xAB).all()
    assert gc.tobytes() == wc.tobytes()
    return got, gc


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(hand_cases()))
def test_device_hand_built(rx, name):
    w, r, c, d, fx, nd, exp = hand_cases()[name]
    got, gc = _same_as_model(rx, w, r, c, d, fx, nd)
    _check(got, gc, exp, d)


def _tapped(rx, iq, segs, mw, scale=None):
    """decode_capture with the tap: host (windows [nseg, mw, L], recs, counts)"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    kw = dict(scale=scale) if scale is not None else {}
    tap, res, cnt = rx._decode_tapped(iq, segs, mw, **kw) if kw else rx._decode_tapped(iq, segs, mw, capi.SC16_SCALE)
    torch.cuda.synchronize()
    recs, counts = capi.results_to_numpy(res, cnt, mw)
    return tap.cpu().numpy().reshape(counts.size, mw, rx.len_epc), recs, counts


@pytest.mark.gpu
def test_device_on_the_recording(rx, cfg1_iq):
    from gen2_uhf_rfid_reader_b200 import capi
    iq = _upload(cfg1_iq)
    whole = abi.make_segments([0], [cfg1_iq.size])
    segs, _, _ = rx.ingest_capture_host(cfg1_iq, max_windows=4)
    assert segs.size == 72
    for table_, mw in ((whole, 160), (segs, 4)):
        w, r, c = _tapped(rx, iq, capi.segments_to_device(table_, "cuda"), mw)
        ok = (r["kind"] == abi.EPC) & (r["crc_ok"] == 1)
        d = np.concatenate([r[ok][:1]["bits"], synth.make_epc_frames(np.arange(24, dtype=np.uint8).reshape(2, 12))])
        got, gc = _same_as_model(rx, w, r, c, d)
        st = got["status"][np.arange(mw)[None, :] < np.minimum(c, mw)[:, None]]
        assert (st == mm.ALREADY_READ).sum() == 70 and (st == mm.MATCHED).sum() == 0


def _truth_frames(n_tags, seed):
    """the simulator's tag frames (synth.make_capture's EPC table)"""
    epc = np.zeros((n_tags, 12), dtype=np.uint8)
    for k in range(n_tags):
        t = np.random.Generator(np.random.Philox(key=[seed + 2, k]))
        epc[k] = t.integers(0, 256, size=12)
        epc[k, 11] = (0x27 + k) & 0xFF
    return synth.make_epc_frames(epc)


WEAK = [(1, 0, 77, 600), (8, 4, 78, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("g", [0.004, 0.003, 0.0025])
@pytest.mark.parametrize("n_tags,q,seed,nseg", WEAK, ids=["1tag", "8tags-q4"])
def test_device_weak_tags(rx, n_tags, q, seed, nseg, g):
    """make_capture weak tags with the truth frames (and random others) as the dictionary, with the recovery records:
    equal to the restatement; no MATCHED window names a tag other than the one that replied, and none is in an empty
    slot"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = capi.Gen2Rx(fixed_q=q)
    cap = synth.make_capture(nseg, device="cpu", seed=seed, fixed_q=q, n_tags=n_tags, tag_gain=g)
    segs = capi.segments_to_device(cap["segments"], "cuda")
    tap, res, cnt = rxq._decode_tapped(_upload(cap["iq"].numpy()), segs, 2, capi.SC16_SCALE)
    qual = rxq.window_quality(tap, res, cnt, 2)
    fix = rxq.recover_epc(tap, res, cnt, qual, 2)
    torch.cuda.synchronize()
    recs, counts = capi.results_to_numpy(res, cnt, 2)
    fx, _ = capi.fixes_to_numpy(fix, cnt, 2)
    w = tap.cpu().numpy().reshape(nseg, 2, rxq.len_epc)
    frames = _truth_frames(n_tags, seed)
    d = np.concatenate([frames, synth.make_epc_frames(np.random.default_rng(5).integers(0, 256, (61, 12)).astype(
        np.uint8))])
    got, gc = _same_as_model(rxq, w, recs, counts, d, fixes=fx)
    st = got[:, 1]["status"]
    matched = st == mm.MATCHED
    truth = cap["truth"]
    assert (truth["n_replies"][matched] > 0).all()
    assert (d[got[matched, 1]["entry"]] == truth["epc"][matched]).all()
    read = int((recs[:, 1]["crc_ok"] == 1).sum())
    rec = int((fx[:, 1]["status"] == abi.FIX_RECOVERED).sum())
    print("%d tags at %g: %d read, %d recovered, %d matched, %d ambiguous, %d no match" % (
        n_tags, g, read, rec, int(matched.sum()), int((st == mm.AMBIGUOUS).sum()), int((st == mm.NO_MATCH).sum())))
    if n_tags == 1 and g == 0.003:
        assert read + rec == 502 and read + rec + int(matched.sum()) > 502


@pytest.mark.gpu
def test_device_on_an_sc16_copy(rx):
    """the weak-tag capture quantised to sc16: decode_capture_match against the report's own tags equals the
    restatement"""
    from gen2_uhf_rfid_reader_b200 import capi
    from test_sc16 import SCALES, quantise
    cap = synth.make_capture(256, device="cpu", tag_gain=0.003, seed=77)
    q16 = _upload(quantise(cap["iq"].numpy(), SCALES[0]))
    segs = capi.segments_to_device(cap["segments"], "cuda")
    out = rx.decode_capture_match(q16, segs, max_windows=2, reject_empty=False, scale=SCALES[0])
    res, cnt, _, fix, tags, summary, _, match, mc = out
    t, sm = capi.tags_to_numpy(tags, summary)
    assert int(sm["n_tags"]) == 1
    got, gcnt = capi.matches_to_numpy(match, cnt, 2, mc)
    w, r, c = _tapped(rx, q16, segs, 2, scale=SCALES[0])
    fx, _ = capi.fixes_to_numpy(fix, cnt, 2)
    want, wc = mm.match(w, r, c, tags.cpu().numpy()[:, :16], fixes=fx, n_dict=int(sm["n_tags"]))
    assert got.tobytes() == want.tobytes() and gcnt.tobytes() == wc.tobytes()
    assert int(gcnt["matched"][0]) > 0
    table_ = capi.tag_table(t, matched=gcnt["matched"])
    assert table_["matched"][0] == gcnt["matched"][0]


@pytest.mark.gpu
def test_device_large_adversarial_dictionary(rx):
    """2,000 slots of 8 weak tags against 30,011 random frames, the 8 true frames and 40 CRC-valid decoys at sign
    distance 4..16 from them: N and K are multiples of no tile size; equal to the restatement"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = capi.Gen2Rx(fixed_q=4)
    cap = synth.make_capture(2000, device="cuda", seed=78, fixed_q=4, n_tags=8, tag_gain=0.003)
    segs = capi.segments_to_device(cap["segments"], "cuda")
    tap, res, cnt = rxq._decode_tapped(cap["iq"], segs, 2, capi.SC16_SCALE)
    torch.cuda.synchronize()
    recs, counts = capi.results_to_numpy(res, cnt, 2)
    w = tap.cpu().numpy().reshape(2000, 2, rxq.len_epc)
    rng = np.random.default_rng(17)
    frames = _truth_frames(8, 78)
    dec = np.concatenate([mm.decoys(f, 5, rng)[0] for f in frames])
    rand = synth.make_epc_frames(rng.integers(0, 256, (30011, 12)).astype(np.uint8))
    d = np.concatenate([rand[:15000], dec, frames, rand[15000:]])
    attempted = (counts == 2) & (recs[:, 1]["kind"] == abi.EPC) & (recs[:, 1]["crc_ok"] == 0)
    if attempted.sum() % 16 == 0:   # leave one EPC window unstored, so the rows fill no tile
        counts[np.nonzero(attempted)[0][0]] = 1
    n_rows = int((attempted & (counts == 2)).sum())
    assert n_rows % 16 and d.shape[0] % 8
    got, gc = _same_as_model(rxq, w, recs, counts, d)
    print("adversarial: %d rows, K = %d, statuses %s" % (n_rows, d.shape[0],
                                                          np.bincount(got[counts == 2, 1]["status"], minlength=6).tolist()))


@pytest.mark.gpu
def test_match_epc_argument_checks(rx):
    """NULL pointers, negative sizes, nseg * max_windows >= 2^31, max_dict > 2^24, a misaligned dictionary, non-finite
    or negative parameters: RFID_B200_EINVAL and nothing written"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    tap = torch.zeros(2 * rx.len_epc, dtype=torch.complex64, device="cuda")
    res = torch.zeros((2, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    dic = torch.zeros((4, 16), dtype=torch.uint8, device="cuda")
    out = torch.zeros((2, 32), dtype=torch.uint8, device="cuda")

    def call(w=tap.data_ptr(), r=res.data_ptr(), c=cnt.data_ptr(), d=dic.data_ptr(), o=out.data_ptr(), n=1, m=2, k=4,
             p=None):
        return L.rfid_b200_match_epc(rx.h, w, r, c, None, n, m, d, None, k, p, o, None, None)

    assert call() == abi.OK and call(n=0) == abi.OK and call(k=0, d=None) == abi.OK
    bad = [dict(w=None), dict(r=None), dict(c=None), dict(o=None), dict(d=None), dict(n=-1), dict(m=-1), dict(k=-1),
           dict(k=(1 << 24) + 1), dict(n=1 << 16, m=1 << 15), dict(d=dic.data_ptr() + 4)]
    for kw in bad:
        assert call(**kw) == abi.EINVAL, kw
    for kw in (dict(max_cost=float("nan")), dict(max_cost=-1.0), dict(min_margin=float("inf")),
               dict(min_margin=-0.5)):
        assert call(p=C.byref(capi.default_match_params(**kw))) == abi.EINVAL, kw
    torch.cuda.synchronize()
    assert (out == 0).all()
