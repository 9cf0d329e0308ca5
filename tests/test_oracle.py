"""CPU tests: the oracle is pinned to the reference's golden vectors and to the reference's own code.

Golden material (SURVEY.md section 4 / Appendix B): README.md:46-53 expected output, the RN16s the reference
author's run decoded (recovered from misc/data/file_sink), and what oracle/_ref (the reference's own blocks under
our scheduler) produced, stored by tests/golden/make_golden.py.
"""
import json
import os
import re
import sys

import numpy as np
import pytest

from conftest import GOLDEN, records_equal
from gen2_uhf_rfid_reader_b200 import abi, synth

sys.path.insert(0, GOLDEN)
from make_golden import RATE_VARIANTS, rate_capture, rate_cases  # noqa: E402
import rate_rule  # noqa: E402


def _readme_numbers():
    txt = open(os.path.join(GOLDEN, "readme_expected.txt")).read()
    g = lambda pat: re.search(pat, txt).group(1)  # noqa: E731
    return {"sent": int(g(r"queryreps sent : (\d+)")), "round": int(g(r"Inventory round : (\d+)")),
            "epc": int(g(r"decoded EPC : (\d+)")), "unique": int(g(r"unique tags : (\d+)")),
            "tag": int(g(r"Tag ID : (\w+)"), 16), "reads": int(g(r"Num of reads : (\d+)"))}


def test_reference_reproduces_readme():
    """the compiled reference + our scheduler print the README block (README.md:48-53)"""
    exp = _readme_numbers()
    t = json.load(open(os.path.join(GOLDEN, "cfg1_ref_stats.json")))["text"]
    assert "queryreps sent : %d" % exp["sent"] in t
    assert "Inventory round : %d" % exp["round"] in t
    assert "decoded EPC : %d" % exp["epc"] in t
    assert "unique tags : %d" % exp["unique"] in t
    assert "Tag ID : %x  Num of reads : %d" % (exp["tag"], exp["reads"]) in t
    assert exp == {"sent": 71, "round": 72, "epc": 70, "unique": 1, "tag": 0x27, "reads": 70}


def test_reference_chunk_size_independent(ref_outputs, cfg1_golden):
    for chunk in (257, 4096, 100000):
        assert not records_equal(ref_outputs["cfg1_records_chunk%d" % chunk], cfg1_golden), chunk


def test_golden_rn16_match_author_run(cfg1_golden):
    """the 71 RN16s decoded on file_source_test are the ones ACKed in the author's TX file misc/data/file_sink"""
    cmds = json.load(open(os.path.join(GOLDEN, "file_sink_commands.json")))
    assert len(cmds["queries"]) == 72 and len(cmds["acks"]) == 71
    assert set(cmds["queries"]) == {"1000000000000000010000"}
    rn = [abi.bits_hex(r) for r in cfg1_golden if r["kind"] == abi.RN16]
    assert rn == cmds["rn16"]
    assert all(a.startswith("01") for a in cmds["acks"])


def test_reference_tx_matches_author_run(ref_outputs):
    """the reader block's own TX envelope (driven by our scheduler) = the committed file_sink, command by command"""
    import sys
    sys.path.insert(0, GOLDEN)
    from make_golden import decode_pie
    tx = ref_outputs["cfg1_tx"]
    cmds = decode_pie(tx)
    gold = json.load(open(os.path.join(GOLDEN, "file_sink_commands.json")))
    q = [b for k, b in cmds if k == "preamble"]
    a = [b for k, b in cmds if k == "framesync"]
    assert q[:72] == gold["queries"] and a[:71] == gold["acks"]
    assert abs(len(tx) - 539864) <= 8  # flowgraph stop point differs by a few samples


def test_restatement_equals_reference_on_cfg1(oracle, cfg1_iq, cfg1_golden):
    recs, n = oracle.decode_stream(cfg1_iq)
    assert n == 142
    assert not records_equal(recs, cfg1_golden)
    # facts recorded in SURVEY.md 8(c)
    assert list(recs["open_index"][:4]) == [7393, 8731, 11302, 12123] and recs["open_index"][-1] == 246811
    epc = [abi.bits_hex(r) for r in recs if r["kind"] == abi.EPC and r["crc_ok"] == 1]
    assert len(epc) == 70 and set(epc) == {"3000300833b2ddd90140000000276d3e"}
    assert recs[1]["crc_ok"] == 0  # the one failed round: late ACK


def test_stats_reduction_matches_reference(oracle, cfg1_golden):
    st = oracle.reduce_stats(cfg1_golden[None, :], np.array([len(cfg1_golden)]), True)
    g = json.load(open(os.path.join(GOLDEN, "cfg1_ref_stats.json")))
    assert (st.n_queries_sent, st.cur_inventory_round, st.cur_slot_number, st.n_epc_correct) == \
        (g["n_queries_sent"], g["cur_inventory_round"], g["cur_slot_number"], g["n_epc_correct"])
    assert st.tag_map() == {int(k): v for k, v in g["tag_reads"].items()}
    from oracle.pyoracle import Oracle
    q4 = np.load(os.path.join(GOLDEN, "cfg1_q4_ref_records.npy"))
    g4 = json.load(open(os.path.join(GOLDEN, "cfg1_q4_ref_stats.json")))
    st4 = Oracle(fixed_q=4).reduce_stats(q4[None, :], np.array([len(q4)]), True)
    assert (st4.n_queries_sent, st4.cur_inventory_round, st4.cur_slot_number, st4.n_epc_correct) == \
        (g4["n_queries_sent"], g4["cur_inventory_round"], g4["cur_slot_number"], g4["n_epc_correct"])


SYNTH_KW = [dict(n_tags=1), dict(n_tags=0), dict(n_tags=6, fixed_q=2), dict(n_tags=1, noise_sigma=0.02)]


@pytest.mark.parametrize("kw", SYNTH_KW)
def test_restatement_equals_reference_on_synthetic(oracle, ref_outputs, kw):
    cap = synth.make_capture(48, seed=21, **kw)
    iq = cap["iq"].numpy()
    i = SYNTH_KW.index(kw)   # same order as make_golden.SYNTH_KW
    rr, rc = ref_outputs["synth48_%d_records" % i], ref_outputs["synth48_%d_counts" % i]
    orr, oc, _ = oracle.decode_segments(iq, cap["segments"], max_per_seg=4)
    assert (rc == oc).all()
    assert not records_equal(rr, orr)
    if kw.get("n_tags") == 1 and "noise_sigma" not in kw:
        assert (rr[:, 0]["tag_id"] == cap["truth"]["rn16"]).all()
        assert (rr[:, 1]["crc_ok"] == 1).all()


def test_mf_order_does_not_change_decisions(oracle, cfg1_iq):
    """matched-filter summation order is unpinned by the reference; decode results do not depend on it"""
    outs = [oracle.decode_decimated(oracle.mf(cfg1_iq, v))[0] for v in (0, 1, 2)]
    for o in outs[1:]:
        for f in ("open_index", "sync_index", "T", "crc_ok", "tag_id", "bits"):
            assert o[f].tobytes() == outs[0][f].tobytes(), f
        assert np.max(np.abs(o["score"] - outs[0]["score"]) / outs[0]["score"]) < 2e-4


def test_blocked_matched_filter_is_the_canonical_one(oracle):
    """The CPU reference arm of bench.py times the canonical boxcar with every block sum formed once (variant 3):
    it must be the canonical order bit for bit, for any length and tap count"""
    rng = np.random.default_rng(5)
    for n in (0, 3, 5, 24, 25, 26, 777, 16960, 16963):
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        assert oracle.mf(x, 0).tobytes() == oracle.mf(x, 3).tobytes(), n
    from oracle.pyoracle import Oracle
    for adc, ntaps in ((1000000, 12), (1000000, 13), (4000000, 50)):
        o = Oracle(adc_rate=adc, ntaps=ntaps)
        x = (rng.standard_normal(5000) + 1j * rng.standard_normal(5000)).astype(np.complex64)
        assert o.mf(x, 0).tobytes() == o.mf(x, 3).tobytes(), (adc, ntaps)


def test_independent_segments_have_their_own_stop_rule():
    """continuous=0: a segment is a reference run with fresh blocks and reader_state, so the unique-tag stop rule
    (gate_impl.cc:101-104) sees only the segment's own tags; the global tag map is for reporting only"""
    from gen2_uhf_rfid_reader_b200 import abi
    from oracle.pyoracle import Oracle
    o = Oracle(max_tags=1)
    recs = np.zeros((3, 4), dtype=abi.RESULT_DTYPE)
    for s in range(3):
        for k in range(4):
            recs[s, k]["kind"] = k & 1
            recs[s, k]["crc_ok"] = 1 if k & 1 else -1
            recs[s, k]["tag_id"] = 10 * s + k      # every EPC a different tag: 2 per segment, 6 globally
    counts = np.full(3, 4, dtype=np.int32)
    st = o.reduce_stats(recs, counts, False)
    # per segment: 2 EPC windows, the second one makes 2 unique tags > max_tags = 1 -> stop AFTER it; all 12 windows count
    assert st.n_windows == 12 and st.n_epc_correct == 6 and st.n_unique_tags == 6
    st_c = o.reduce_stats(recs, counts, True)
    # one continuous run: stops after the second unique tag, i.e. after 4 windows
    assert st_c.n_windows == 4 and st_c.n_epc_correct == 2


def test_crc_known_answers(oracle):
    assert oracle.query_bits(0) == "1000000000000000010000"   # file_sink content / SURVEY Appendix B
    assert oracle.query_bits(4) == "1000000000000010011101"
    assert "".join(map(str, synth.query_bits(0))) == oracle.query_bits(0)
    assert "".join(map(str, synth.query_bits(4))) == oracle.query_bits(4)
    frame = bytes.fromhex("3000300833b2ddd90140000000276d3e")  # the recorded tag's PC+EPC+CRC
    assert oracle.crc16(frame[:14]) == 0x6D3E and oracle.crc16_ok(frame) == 1
    assert synth.crc16_gen2(frame[:14]) == 0x6D3E
    bad = bytearray(frame)
    bad[5] ^= 1
    assert oracle.crc16_ok(bytes(bad)) == 0


def test_cabsf_is_double_sqrt(oracle):
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(20000) * 10 ** rng.uniform(-3, 2, 20000)).astype(np.float32)
    y = (rng.standard_normal(20000) * 10 ** rng.uniform(-3, 2, 20000)).astype(np.float32)
    want = np.sqrt(x.astype(np.float64) ** 2 + y.astype(np.float64) ** 2).astype(np.float32)
    got = np.array([oracle.cabsf(float(a), float(b)) for a, b in zip(x, y)], dtype=np.float32)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("adc,exp", [(1000000, (5, 5.0, 48, 2, 50, 24, 125, 685)), (2000000, (10, 10.0, 96, 4, 100, 48, 250, 1370)),
                                     (4000000, (20, 20.0, 192, 9, 200, 96, 500, 2740)), (6000000, (30, 30.0, 288, 14, 300, 144, 750, 4110)),
                                     (8000000, (40, 40.0, 384, 19, 400, 192, 1000, 5480))])
def test_rate_sweep_derived_counts(adc, exp):
    """SURVEY.md Appendix A.6 (evaluated there with the reference's own expressions)"""
    from oracle.pyoracle import Oracle
    c = Oracle(adc_rate=adc).cfg
    assert (c.n_tag_bit_i, c.n_tag_bit_f, c.n_T1, c.n_PW, c.win_length, c.dc_length, c.len_rn16, c.len_epc) == exp


def test_empty_and_short_segments(oracle):
    cap = synth.make_capture(2, seed=1)
    iq = cap["iq"].numpy()
    segs = abi.make_segments([0, 5, 100, 0], [0, 3, 4, 700])
    recs, counts, _ = oracle.decode_segments(iq, segs, max_per_seg=2)
    assert counts.tolist() == [0, 0, 0, 0]


# ------------------------------------------------------------------ other sample rates
@pytest.fixture(scope="session")
def ref_rates():
    """What the reference's own blocks computed at other sample rates (tests/golden/make_golden.py: rate_outputs)."""
    with np.load(os.path.join(GOLDEN, "reference_rates.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("case", rate_cases(), ids=[c[0] for c in rate_cases()])
def test_restatement_equals_reference_at_other_rates(ref_rates, case):
    """the restatement against the reference's compiled blocks at every stored rate, tap count and capture variant,
    every field of every record and the window counts"""
    from oracle.pyoracle import Oracle
    key, adc, ntaps, kw = case
    cap = rate_capture(adc, kw)
    orr, oc, _ = Oracle(adc_rate=adc, ntaps=ntaps, fixed_q=kw.get("fixed_q", 0)).decode_segments(
        cap["iq"].numpy(), cap["segments"], max_per_seg=4)
    assert oc.tolist() == ref_rates[key + "_counts"].tolist()
    assert not records_equal(orr, ref_rates[key + "_records"])
    assert oc.sum() >= 8


def _sync_correlation(win, n):
    """tag_sync's |corr|^2 for every i < 1.5 n (tag_decoder_impl.cc:85-95), float32 in the reference's order"""
    i = np.arange(int(np.ceil(1.5 * float(n))))
    cr, ci = np.zeros(i.size, np.float32), np.zeros(i.size, np.float32)
    for j, p in enumerate((1, 1, 0, 1, 0, 0, 1, 0, 0, 0, 1, 1)):
        k = (i.astype(np.float32) + np.float32(j) * n / np.float32(2)).astype(np.int64)
        if p:
            cr, ci = cr + win[k].real, ci + win[k].imag
    return cr * cr + ci * ci


def _period_energies(win, n, index):
    """tag_detection_EPC's energy[t] and half-periods (tag_decoder_impl.cc:151-166), float32 in the reference's order"""
    n64 = np.float64(n)
    lo, hi = np.float32(n64 / 2.0 - n64 / 2.0 / 100), np.float32(n64 / 2.0 + n64 / 2.0 / 100)
    steps = lo + np.arange(20, dtype=np.float32) * (hi - lo) / np.float32(19)
    m2 = win.real * win.real + win.imag * win.imag
    e = np.zeros(20, np.float32)
    for q in range(256):
        e = e + m2[(np.float32(q) * steps + np.float32(index)).astype(np.int64)]
    return e, steps


def test_quiet_captures_tie_the_first_maximum_rules():
    """The noise- and drift-free captures of the rate comparisons exist to produce exact ties where the reference keeps
    the first maximum (tag_sync's strict '>', std::max_element).  Recompute both searches in numpy float32 on the
    gate's windows: the first maximum is the restatement's sync_index and T, and ties do occur, in both searches."""
    from oracle.pyoracle import Oracle
    sync_ties, t_ties = {}, {}
    for key, adc, ntaps, kw in rate_cases():
        if kw is not RATE_VARIANTS["quiet"]:
            continue
        o = Oracle(adc_rate=adc, ntaps=ntaps)
        n = np.float32(o.cfg.n_tag_bit_f)
        cap = rate_capture(adc, kw)
        iq = cap["iq"].numpy()
        sync_ties[adc, ntaps] = t_ties[adc, ntaps] = 0
        for s in cap["segments"]:
            y = o.mf(iq[int(s["offset"]):int(s["offset"]) + int(s["length"])])
            wins = o.gate(y, want_windows=True)["windows"]
            recs, _ = o.decode_decimated(y)
            for k, r in enumerate(recs):
                w = wins[k, :r["length"]]
                c = _sync_correlation(w, n)
                first = int(np.argmax(c))
                assert first == r["sync_index"] and c[first] == r["score"], (key, k)
                sync_ties[adc, ntaps] += int((c == c[first]).sum() > 1)
                if r["kind"] == abi.EPC:
                    index = int(np.float32(first) + np.float32(6) * n + n / np.float32(2))
                    e, steps = _period_energies(w, n, index)
                    t = int(np.argmax(e))
                    assert steps[t] == r["T"], (key, k)
                    t_ties[adc, ntaps] += int((e == e[t]).sum() > 1)
    assert sum(v > 0 for v in sync_ties.values()) >= 4, sync_ties
    assert sum(t_ties.values()) > 0, t_ties


def test_well_defined_rates_restatement_agrees_with_numpy():
    """gen2_oracle_make_cfg's `defined` against the independent numpy evaluation, on the 1 kHz grid from 1 to 8 MS/s;
    the restatement refuses an undefined configuration instead of reading past its window"""
    from oracle.pyoracle import Oracle, derive_cfg
    want = rate_rule.well_defined(rate_rule.GRID)
    got = np.array([derive_cfg(adc_rate=int(r)).defined for r in rate_rule.GRID], dtype=bool)
    assert (got == want).all(), rate_rule.GRID[got != want][:10]
    assert int(want.sum()) == 314
    for adc, ntaps in {(a, t) for _, a, t, _ in rate_cases()}:
        assert want[rate_rule.GRID == adc].all(), adc
    for adc in (1_360_000, 1_520_000, 2_500_000, 5_800_000):
        assert not rate_rule.well_defined(np.array([adc]))[0]
    with pytest.raises(ValueError, match="past the end"):
        Oracle(adc_rate=1_360_000)
    with pytest.raises(ValueError):
        Oracle(adc_rate=1_687_500)
