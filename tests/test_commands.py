"""Capture mode, the reader's side: PIE commands decoded per segment (rfid_b200_decode_commands) and paired with the tag
windows they armed (capi.transcript).

CPU: the numpy restatement of the rule (command_model.py) on the reference's recording, on synthetic slots and on a
hand-built PIE envelope.  GPU: the device records equal the restatement's bit for bit, and decode back what the
simulator and the TX synthesiser sent.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import command_model as cm
import segmenter_model as sm
from conftest import GOLDEN
from gen2_uhf_rfid_reader_b200 import abi, synth

COMMANDS = json.load(open(os.path.join(GOLDEN, "file_sink_commands.json")))


def _table(iq):
    segs, _ = sm.segment_table(iq)
    return abi.make_segments([o for o, _ in segs], [n for _, n in segs])


def _flat(recs, counts):
    return np.concatenate([recs[s, :min(counts[s], recs.shape[1])] for s in range(counts.size)])


def _check_recording(cmds):
    q = cmds[cmds["kind"] == abi.TX_QUERY]
    a = cmds[cmds["kind"] == abi.TX_ACK]
    assert len(cmds) == len(q) + len(a) == 72 + 71
    assert [cm.bits_str(r) for r in q] == COMMANDS["queries"]
    assert (q["crc_ok"] == 1).all() and (q["arg"] == 0).all()
    assert (q["tari"] == 48).all() and (q["rtcal"] == 144).all() and (q["trcal"] == 400).all()
    assert ["%04x" % v for v in a["arg"]] == COMMANDS["rn16"]
    assert [cm.bits_str(r) for r in a] == COMMANDS["acks"]
    assert (a["trcal"] == 0).all() and (a["n_bits"] == 18).all()


# ------------------------------------------------------------------ CPU: the rule
def test_model_on_the_recording_whole_and_segmented(cfg1_iq):
    """72 Queries (Q 0, CRC-5 passing, Tari/RTcal/TRcal = 48/144/400 samples) and 71 ACKs echoing the recorded RN16s,
    nothing else, whether the recording is one segment or the segmenter's 72"""
    whole = cm.decode_segment(cfg1_iq)
    _check_recording(whole)
    segs = _table(cfg1_iq)
    assert segs.size == 72
    recs, counts = cm.decode_segments(cfg1_iq, segs, 8)
    assert counts.tolist() == [2] * 71 + [1]
    flat = _flat(recs, counts)
    _check_recording(flat)
    # the same commands at the same absolute places
    starts = flat["start"].astype(np.int64) + np.repeat(segs["offset"].astype(np.int64), counts)
    assert starts.tolist() == whole["start"].astype(np.int64).tolist()


def test_transcript_of_the_recording(cfg1_iq, cfg1_golden):
    """every RN16 window armed by a Query, every EPC window by the ACK that echoes its RN16; the ACK turnaround of the
    first EPC (the one whose CRC fails) is 1738.5 us, the median 421.5 us"""
    from gen2_uhf_rfid_reader_b200 import capi
    cmds = cm.decode_segment(cfg1_iq)
    t = capi.transcript(cmds[None, :], np.array([cmds.size]), cfg1_golden[None, :], np.array([cfg1_golden.size]), 5)
    assert t.size == 142
    rn16, epc = t[t["kind"] == abi.RN16], t[t["kind"] == abi.EPC]
    assert rn16.size == epc.size == 71
    assert (rn16["cmd_kind"] == abi.TX_QUERY).all() and (rn16["ack_echo"] == -1).all()
    assert np.isnan(rn16["turnaround_us"]).all()
    assert (epc["cmd_kind"] == abi.TX_ACK).all() and (epc["ack_echo"] == 1).all()
    assert rn16["command"].tolist() == list(range(0, 142, 2)) and epc["command"].tolist() == list(range(1, 142, 2))
    ta = epc["turnaround_us"]
    first_epc = cfg1_golden[cfg1_golden["kind"] == abi.EPC][0]
    assert ta[0] == 1738.5 and first_epc["crc_ok"] == 0
    assert np.median(ta) == 421.5
    assert ta.min() == 420.5 and sorted(ta)[-3:] == [422.5, 540.0, 1738.5]
    assert (ta > 500).sum() == 2 and ta.sum() == 31366.5


RATES = (1_000_000, 2_000_000, 4_000_000, 8_000_000)
SYNTH_CASES = [(0, 1), (4, 8)]   # (fixed_q, n_tags)


@pytest.mark.parametrize("adc", RATES, ids=["1M", "2M", "4M", "8M"])
@pytest.mark.parametrize("q,tags", SYNTH_CASES, ids=["q0-1tag", "q4-8tags"])
def test_model_on_synthetic_slots(adc, q, tags):
    """every slot: a Query (slot 0 of a round) or a QueryRep, with Q and the CRC as sent, then the ACK of the RN16"""
    cap = synth.make_capture(12, adc_rate=adc, fixed_q=q, n_tags=tags, seed=77 + q, device="cpu")
    iq = cap["iq"].numpy()
    recs, counts = cm.decode_segments(iq, cap["segments"], 4, adc_rate=adc)
    tr = cap["truth"]
    assert (counts == 2).all()
    first, ack = recs[:, 0], recs[:, 1]
    assert (first["kind"] == np.where(tr["is_query"], abi.TX_QUERY, abi.TX_QUERY_REP)).all()
    isq = tr["is_query"]
    assert (first["arg"][isq] == q).all() and (first["crc_ok"][isq] == 1).all()
    assert (first["arg"][~isq] == 0).all() and (first["crc_ok"][~isq] == -1).all()
    assert [cm.bits_str(r) for r in first[isq]] == ["".join(map(str, synth.query_bits(q)))] * int(isq.sum())
    assert (ack["kind"] == abi.TX_ACK).all() and (ack["arg"] == tr["rn16"]).all()
    sps = adc // 1_000_000
    assert (first["tari"] == 24 * sps).all() and (first["rtcal"] == 72 * sps).all()
    assert (first["trcal"][isq] == 200 * sps).all() and (first["trcal"][~isq] == 0).all()


# A PIE envelope built here from synth.py's durations and the reader's bit layouts (reader_impl.cc:109-162): every
# symbol is its high part followed by a PW low pulse; a delimiter is a PW low pulse of its own.
def _symbols(sync, bits):
    sym = [(0, synth.DELIM_US), (synth.DATA0_US - synth.PW_US, synth.PW_US), (synth.RTCAL_US - synth.PW_US, synth.PW_US)]
    if sync == "preamble":
        sym.append((synth.TRCAL_US - synth.PW_US, synth.PW_US))
    for b in bits:
        d = synth.DATA1_US if b == "1" else synth.DATA0_US
        sym.append((d - synth.PW_US, synth.PW_US))
    return sym


def _pie_capture(script, adc, seed=5):
    """script: ("cw", us) | ("low", us) | (sync, bitstring) -> complex64 capture at adc"""
    lv = []
    for item in script:
        if item[0] == "cw":
            lv += [1.0] * item[1]
        elif item[0] == "low":
            lv += [0.0] * item[1]
        else:
            for hi, lo in _symbols(*item):
                lv += [1.0] * hi + [0.0] * lo
    env = np.repeat(np.array(lv, dtype=np.float64), adc // 1_000_000)
    env = synth.FLOOR + (1.0 - synth.FLOOR) * env
    if adc == 2_000_000:
        fir = np.array(synth.EDGE_FIR_2MSPS)
        env = np.convolve(np.concatenate([np.ones(fir.size - 1), env]), fir, mode="valid")
    rng = np.random.default_rng(seed)
    noise = rng.normal(0, synth.NOISE_SIGMA, size=(env.size, 2)) @ np.array([1, 1j])
    return (synth.LEAK * env + noise).astype(np.complex64)


PIE_SCRIPT = [("cw", 700), ("frame-sync", "11000000"), ("cw", 900), ("frame-sync", "100100000"), ("cw", 2500),
              ("low", 2000), ("cw", 900), ("frame-sync", "101101"), ("cw", 1000), ("preamble", "1000000000000"),
              ("cw", 600), ("frame-sync", "0011"), ("cw", 600), ("frame-sync", "01" + "1011001110001111"), ("cw", 800)]
PIE_WANT = [(abi.TX_NAK, -1, "11000000"), (abi.TX_QUERY_ADJUST, 0, "100100000"), (cm.CMD_OTHER, -1, "101101"),
            (cm.CMD_OTHER, -1, "1000000000000"), (abi.TX_QUERY_REP, 3, "0011"),
            (abi.TX_ACK, 0xB38F, "01" + "1011001110001111")]


@pytest.mark.parametrize("adc", (1_000_000, 2_000_000, 4_000_000), ids=["1M", "2M", "4M"])
def test_model_on_a_pie_envelope(adc):
    """NAK, QueryAdjust, a power-down, carrier-only stretches and unrecognised bit strings decode back to the script;
    the power-down is a stray burst and yields no record"""
    x = _pie_capture(PIE_SCRIPT, adc)
    got = cm.decode_segment(x, adc_rate=adc)
    assert [(int(r["kind"]), int(r["arg"]), cm.bits_str(r)) for r in got] == PIE_WANT
    assert (got["crc_ok"] == -1).all() and got["index"].tolist() == list(range(len(PIE_WANT)))
    sps = adc // 1_000_000
    assert (got["tari"] == 24 * sps).all() and (got["rtcal"] == 72 * sps).all()
    assert got["trcal"].tolist() == [0, 0, 0, 200 * sps, 0, 0]


# ------------------------------------------------------------------ GPU
def _rx(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.Gen2Rx(**kw)


@pytest.fixture(scope="module")
def rx():
    return _rx()


def _device(rx, x, segs, max_commands, params=None, scale=None):
    """decode_commands of host capture x (complex64, or int16 for sc16) with a host segment table"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    iq = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    dsegs = capi.segments_to_device(segs, "cuda")
    kw = {"scale": scale} if scale is not None else {}
    c, n = rx.decode_commands(iq, dsegs, max_commands=max_commands, params=params, **kw)
    torch.cuda.synchronize()
    return capi.commands_to_numpy(c, n, max_commands)


def _params(**kw):
    from gen2_uhf_rfid_reader_b200 import capi
    return capi.default_cmd_params(**kw)


def _same(got, want):
    (g, gn), (w, wn) = got, want
    assert gn.tolist() == wn.tolist()
    assert g.tobytes() == w.tobytes()


@pytest.mark.gpu
def test_device_on_the_recording(rx, cfg1_iq, cfg1_golden):
    """whole, as the segmenter's 72 segments, and as ragged segments that start and end inside commands at odd
    offsets: the restatement's records bit for bit; the device transcript arms every window as on the CPU"""
    from gen2_uhf_rfid_reader_b200 import capi
    whole = abi.make_segments([0], [cfg1_iq.size])
    got = _device(rx, cfg1_iq, whole, 256)
    _same(got, cm.decode_segments(cfg1_iq, whole, 256))
    _check_recording(got[0][0, :got[1][0]])
    host = rx.decode_commands_host(cfg1_iq, whole, max_commands=256)
    _same(host, got)
    segs = _table(cfg1_iq)
    got = _device(rx, cfg1_iq, segs, 4)
    _same(got, cm.decode_segments(cfg1_iq, segs, 4))
    recs, counts = rx.decode_capture_host(cfg1_iq, segs, max_windows=4)
    t = capi.transcript(got[0], got[1], recs, counts, 5)
    assert t.size == 142
    assert (t["cmd_kind"] == np.where(t["kind"] == abi.RN16, abi.TX_QUERY, abi.TX_ACK)).all()
    assert (t[t["kind"] == abi.EPC]["ack_echo"] == 1).all()
    rng = np.random.default_rng(11)
    starts = cm.decode_segment(cfg1_iq)["start"]
    offs = [int(s) + int(d) for s, d in zip(starts[::3], rng.integers(1, 400, size=starts[::3].size))]
    offs = [o | 1 for o in offs]
    lens = [int(v) for v in rng.integers(300, 30000, size=len(offs))]
    offs += [cfg1_iq.size - 5001, cfg1_iq.size - 1]
    lens += [5001, 1]
    rag = abi.make_segments(offs, lens)
    got = _device(rx, cfg1_iq, rag, 3)
    want = cm.decode_segments(cfg1_iq, rag, 3)
    _same(got, want)
    assert (want[1] > 0).sum() > 10 and (want[1] > 3).any()


@pytest.mark.gpu
def test_device_edge_segments_overflow_and_level_abs(rx, cfg1_iq):
    """empty, 1-sample and command-free segments; more commands than max_commands (counts complete, the leading
    records stored; max_commands 0 counts only); an absolute level"""
    cmds = cm.decode_segment(cfg1_iq)
    quiet = int(cmds["end"][0]) + 11, int(cmds["start"][1]) - int(cmds["end"][0]) - 20   # carrier and the RN16 reply
    segs = abi.make_segments([0, 5, quiet[0], 7, 4001, 0], [0, 1, quiet[1], 2, 1, 1])
    got = _device(rx, cfg1_iq, segs, 2)
    _same(got, cm.decode_segments(cfg1_iq, segs, 2))
    assert got[1].tolist() == [0] * 6
    whole = abi.make_segments([0, 0], [cfg1_iq.size, 200000])
    full = cm.decode_segments(cfg1_iq, whole, 256)
    for m in (1, 5):
        got = _device(rx, cfg1_iq, whole, m)
        assert got[1].tolist() == full[1].tolist() and got[1][0] == 143
        assert got[0].tobytes() == np.ascontiguousarray(full[0][:, :m]).tobytes()
    _, n0 = _device(rx, cfg1_iq, whole, 0)
    assert n0.tolist() == full[1].tolist()
    segs = _table(cfg1_iq)
    for la in (0.05, 0.12):
        got = _device(rx, cfg1_iq, segs, 4, params=_params(level_abs=la))
        _same(got, cm.decode_segments(cfg1_iq, segs, 4, level_abs=la))
    # 0.12 (0.42 of the carrier amplitude) reads the recording's commands; 0.05 also takes the noise of the recording's
    # quiet first 12 ms for a burst
    got = _flat(*_device(rx, cfg1_iq, segs, 4, params=_params(level_abs=0.12)))
    _check_recording(got)
    got = _flat(*_device(rx, cfg1_iq, segs, 4, params=_params(level_abs=0.05)))
    assert got["kind"].tolist() == [cm.CMD_OTHER] + [abi.TX_QUERY, abi.TX_ACK] * 71 + [abi.TX_QUERY]


SIM_CASES = [(0, 1), (2, 4), (4, 8)]   # (fixed_q, n_tags)


@pytest.mark.gpu
@pytest.mark.parametrize("adc", RATES, ids=["1M", "2M", "4M", "8M"])
@pytest.mark.parametrize("q,tags", SIM_CASES, ids=["q0-1tag", "q2-4tags", "q4-8tags"])
def test_device_on_simulated_slots(adc, q, tags):
    """closed-loop simulator slots: a Query iff the slot opens a round (else a QueryRep), Q as configured with a
    passing CRC-5, and an ACK iff the reader sent one, echoing the RN16 it decoded; the first slots equal the
    restatement bit for bit"""
    from gen2_uhf_rfid_reader_b200 import capi
    rxq = _rx(adc_rate=adc, ntaps=max(12, adc // 80000), fixed_q=q)
    sim = capi.default_sim(n_tags=tags, closed_loop=1, seed=900 + q)
    nseg = 48
    cap = rxq.sim_capture(sim, nseg)
    c, n = rxq.decode_commands(cap["iq"], cap["segs"], max_commands=4)
    cmds, counts = capi.commands_to_numpy(c, n, 4)
    truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
    acked = truth["acked_rn16"] >= 0
    assert counts.tolist() == (1 + acked).tolist()
    first = cmds[:, 0]
    isq = truth["is_query"] == 1
    assert (first["kind"] == np.where(isq, abi.TX_QUERY, abi.TX_QUERY_REP)).all()
    assert (first["arg"][isq] == q).all() and (first["crc_ok"][isq] == 1).all()
    assert (cmds[acked, 1]["kind"] == abi.TX_ACK).all() and (cmds[acked, 1]["arg"] == truth["acked_rn16"][acked]).all()
    assert isq.any() and acked.any()
    if q > 0:
        assert (~isq).any()
    k = 6
    iq = cap["iq"][:k * cap["segment_len"]].cpu().numpy()
    segs = cap["segs"][:k].cpu().numpy().view(abi.SEGMENT_DTYPE).reshape(-1)
    want = cm.decode_segments(iq, segs, 4, adc_rate=adc)
    assert counts[:k].tolist() == want[1].tolist()
    assert cmds[:k].tobytes() == want[0].tobytes()


def _synth_capture(rx, script, adc=2_000_000, dac=1_000_000, seed=3):
    """tx_synth waveform held to the ADC rate, with carrier leakage and noise -> host complex64"""
    import torch
    tx = rx.tx_synth(script, dac_rate=dac)
    env = torch.repeat_interleave(tx, adc // dac).double()
    env = synth.FLOOR + (1.0 - synth.FLOOR) * env
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    noise = torch.randn(env.numel(), 2, generator=g, device="cuda", dtype=torch.float64) * synth.NOISE_SIGMA
    x = torch.complex(synth.LEAK.real * env + noise[:, 0], synth.LEAK.imag * env + noise[:, 1]).to(torch.complex64)
    return x.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("q", (0, 5))
def test_device_decodes_tx_synth_scripts(q):
    """Query, QueryRep, ACK, NAK and QueryAdjust, each followed by carrier, decode back to the script; a power-down with
    carrier around it is a stray burst"""
    rxq = _rx(fixed_q=q)
    T = abi
    script = [(T.TX_START, 0), (T.TX_QUERY, 0), (T.TX_CW, 0), (T.TX_QUERY_REP, 0), (T.TX_CW, 0), (T.TX_ACK, 0x5A3C),
              (T.TX_CW, 0), (T.TX_NAK, 0), (T.TX_CW, 0), (T.TX_QUERY_ADJUST, 0), (T.TX_CW, 0), (T.TX_POWER_DOWN, 0),
              (T.TX_START, 0), (T.TX_ACK, 0x0001), (T.TX_CW, 0)]
    x = _synth_capture(rxq, script)
    segs = abi.make_segments([0], [x.size])
    got = _device(rxq, x, segs, 16)
    _same(got, cm.decode_segments(x, segs, 16))
    r = got[0][0, :got[1][0]]
    assert [(int(k), int(a)) for k, a in zip(r["kind"], r["arg"])] == [
        (T.TX_QUERY, q), (T.TX_QUERY_REP, 0), (T.TX_ACK, 0x5A3C), (T.TX_NAK, -1), (T.TX_QUERY_ADJUST, 0),
        (T.TX_ACK, 0x0001)]
    assert r["crc_ok"].tolist() == [1, -1, -1, -1, -1, -1]
    assert cm.bits_str(r[0]) == "".join(map(str, synth.query_bits(q)))


@pytest.mark.gpu
def test_device_nak_then_query_and_the_gap():
    """a NAK is followed by only 250 us of carrier: with gap_us 220 it and the next Query are two commands, at the
    default gap one OTHER burst"""
    rx0 = _rx()
    T = abi
    x = _synth_capture(rx0, [(T.TX_START, 0), (T.TX_NAK, 0), (T.TX_QUERY, 0), (T.TX_CW, 0)])
    segs = abi.make_segments([0], [x.size])
    got = _device(rx0, x, segs, 4, params=_params(gap_us=220))
    _same(got, cm.decode_segments(x, segs, 4, gap_us=220))
    assert got[0][0, :got[1][0]]["kind"].tolist() == [T.TX_NAK, T.TX_QUERY]
    got = _device(rx0, x, segs, 4)
    _same(got, cm.decode_segments(x, segs, 4))
    assert got[0][0, :got[1][0]]["kind"].tolist() == [cm.CMD_OTHER]


@pytest.mark.gpu
def test_device_sc16_equals_fc32(rx, cfg1_iq):
    """int16 recording: records of the fc32 conversion (device and _host) at every segment offset residue mod 4"""
    from test_sc16 import SCALES, convert, quantise
    scale = SCALES[0]
    q = quantise(cfg1_iq, scale)
    x = convert(q, scale)
    base = _table(cfg1_iq)
    for r in range(4):
        segs = base.copy()
        segs["offset"] = segs["offset"] + np.uint64(r)
        segs["length"] = segs["length"] - np.uint32(r + 3)
        segs = np.concatenate([segs, abi.make_segments([x.size - 7 + r], [7 - r])])
        got = _device(rx, q, segs, 4, scale=scale)
        _same(got, _device(rx, x, segs, 4))
        _same(got, rx.decode_commands_host(x, segs, max_commands=4))
        _same(got, cm.decode_segments(x, segs, 4))
        assert got[1][:71].tolist() == [2] * 71


@pytest.mark.gpu
def test_decode_capture_unchanged_around_decode_commands(cfg1_iq):
    """decode_capture records and counts are the same when decode_commands runs before and after it on the same
    stream and context"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    segs = _table(cfg1_iq)
    iq = torch.from_numpy(cfg1_iq.copy()).cuda()
    dsegs = capi.segments_to_device(segs, "cuda")
    ref = capi.results_to_numpy(*_rx().decode_capture(iq, dsegs, max_windows=4), 4)
    rx1 = _rx()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        c0 = rx1.decode_commands(iq, dsegs, max_commands=4, stream=s)
        r = rx1.decode_capture(iq, dsegs, max_windows=4, stream=s)
        c1 = rx1.decode_commands(iq, dsegs, max_commands=4, stream=s)
    s.synchronize()
    got = capi.results_to_numpy(*r, 4)
    assert got[1].tolist() == ref[1].tolist() and got[0].tobytes() == ref[0].tobytes()
    assert capi.commands_to_numpy(*c0, 4)[0].tobytes() == capi.commands_to_numpy(*c1, 4)[0].tobytes()


@pytest.mark.gpu
def test_decode_commands_argument_checks(rx):
    """level_frac outside (0, 1), level_abs negative or not finite, gap_us <= 0, negative counts, NULL pointers, a bad
    sc16 scale or alignment, a misaligned fc32 pointer: RFID_B200_EINVAL; a segment longer than INT32_MAX is EINVAL
    on the host call and a count of RFID_B200_EINVAL on the device call"""
    import torch
    from gen2_uhf_rfid_reader_b200 import capi
    L = capi.load_library()
    x = torch.zeros(4096 + 8, dtype=torch.complex64, device="cuda")
    q = torch.zeros(2 * 4096 + 8, dtype=torch.int16, device="cuda")
    segs = capi.segments_to_device(abi.make_segments([0], [4000]), "cuda")
    out = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    hx = np.zeros(4096, dtype=np.complex64)
    hs = abi.make_segments([0], [4000])
    ho = np.zeros(8, dtype=abi.COMMAND_DTYPE)
    hc = np.zeros(2, dtype=np.int32)

    def dev(p=None, n=1, m=4, ptr=None, o=out):
        return L.rfid_b200_decode_commands(rx.h, ptr or x.data_ptr(), 4096, segs.data_ptr(), n, p, m,
                                           o.data_ptr() if o is not None else None, cnt.data_ptr(), None)

    def host(p=None, n=1, m=4, hsegs=hs):
        return L.rfid_b200_decode_commands_host(rx.h, hx.ctypes.data, 4096, hsegs.ctypes.data, n, p, m, ho.ctypes.data,
                                                hc.ctypes.data)

    bad = [dict(level_frac=0.0), dict(level_frac=1.0), dict(level_frac=-0.5), dict(level_frac=float("nan")),
           dict(level_abs=-1.0), dict(level_abs=float("inf")), dict(level_abs=float("nan")), dict(gap_us=0.0),
           dict(gap_us=-400.0), dict(gap_us=float("nan"))]
    for kw in bad:
        p = C.byref(_params(**kw))
        assert dev(p) == abi.EINVAL and host(p) == abi.EINVAL, kw
        assert L.rfid_b200_decode_commands_sc16(rx.h, q.data_ptr(), 4096, 1.0 / 32767, segs.data_ptr(), 1, p, 4,
                                                out.data_ptr(), cnt.data_ptr(), None) == abi.EINVAL, kw
        with pytest.raises(capi.RfidB200Error):
            rx.decode_commands(x, segs, max_commands=4, params=_params(**kw))
    assert dev(n=-1) == abi.EINVAL and dev(m=-1) == abi.EINVAL and dev(o=None) == abi.EINVAL
    assert host(n=-1) == abi.EINVAL and host(m=-1) == abi.EINVAL
    assert dev(ptr=x.data_ptr() + 4) == abi.EINVAL
    for sc in (0.0, -1.0, float("nan"), float("inf")):
        assert L.rfid_b200_decode_commands_sc16(rx.h, q.data_ptr(), 4096, sc, segs.data_ptr(), 1, None, 4,
                                                out.data_ptr(), cnt.data_ptr(), None) == abi.EINVAL
    for shift in (2, 4, 6):
        assert L.rfid_b200_decode_commands_sc16(rx.h, q.data_ptr() + 2 * shift, 4096, 1.0 / 32767, segs.data_ptr(), 1,
                                                None, 4, out.data_ptr(), cnt.data_ptr(), None) == abi.EINVAL
    assert dev() == 0 and dev(m=0, o=None) == 0 and host() == 0
    huge = abi.make_segments([0, 0], [0x80000000, 100])
    assert host(hsegs=huge, n=2) == abi.EINVAL
    got = _device(rx, hx, huge, 2)
    assert got[1].tolist() == [abi.EINVAL, 0]
    torch.cuda.synchronize()
