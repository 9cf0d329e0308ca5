#!/usr/bin/env python
"""Regenerates tests/golden/* from /root/reference (run in the build container only).

  file_source_test.c64.xz   the reference's recorded RX capture (gr-rfid/misc/data/file_source_test,
                            1,247,958 complex64 @ 2 MS/s), xz-compressed verbatim: the cfg1 parity input
  file_sink_commands.json   Query / ACK bit strings decoded from the reference author's committed TX output
                            gr-rfid/misc/data/file_sink (PIE: data0 = 24 samples fall-to-fall, data1 = 48;
                            reader_impl.cc:51-71,84-125) -- 72 Queries and 71 ACKs whose payloads are the
                            RN16s the reference decoded on that run (SURVEY.md Appendix B)
  readme_expected.txt       the known-answer block of README.md:46-53
  cfg1_ref_records.npy      rfid_b200_window_result records produced by oracle/_ref (the reference's own
                            blocks) on file_source_test; cfg1_ref_stats.json the READER_STATS + print_results text
  cfg1_q4_*.                the same with FIXED_Q = 4
  reference_outputs.npz     everything else the tests compare with the reference's own blocks (see
                            reference_outputs()), so that the suite runs where the reference is absent
  reference_rates.npz       oracle/_ref records and counts at other sample rates (rate_outputs(); regenerate it
                            alone with `make_golden.py rates`)
  reference_pulses.npz      oracle/_ref records and counts on the pulse-train captures (pulse_outputs(); regenerate it
                            alone with `make_golden.py pulses`)
"""
import json
import lzma
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = "/root/reference"


def decode_pie(tx):
    """TX envelope (0/1 floats @1 MS/s) -> list of (kind, bitstring)."""
    lvl = tx > 0.5
    fall = np.nonzero(lvl[:-1] & ~lvl[1:])[0] + 1   # first low sample of each pulse
    # group falls into commands: gaps > 400 samples separate commands
    cmds, cur = [], [fall[0]]
    for a, b in zip(fall[:-1], fall[1:]):
        if b - a > 400:
            cmds.append(cur)
            cur = []
        cur.append(b)
    cmds.append(cur)
    out = []
    for c in cmds:
        d = np.diff(c)
        iv = list(d)
        # fall-to-fall intervals: delimiter->data0 low = 24, RTcal = 72, TRcal = 200 (Query only),
        # then one interval per bit (every PIE symbol ends with its low pulse): 24 = '0', 48 = '1'
        assert iv[0] == 24 and iv[1] == 72, iv[:4]
        k = 2
        kind = "framesync"
        if iv[k] == 200:
            kind = "preamble"
            k += 1
        assert all(x in (24, 48) for x in iv[k:]), iv
        bits = "".join("1" if x == 48 else "0" for x in iv[k:])
        out.append((kind, bits))
    return out


def main():
    src = os.path.join(REF, "gr-rfid/misc/data/file_source_test")
    raw = open(src, "rb").read()
    with open(os.path.join(HERE, "file_source_test.c64.xz"), "wb") as f:
        f.write(lzma.compress(raw, preset=9 | lzma.PRESET_EXTREME))

    sink = np.fromfile(os.path.join(REF, "gr-rfid/misc/data/file_sink"), dtype=np.complex64).real
    amp = sink.max()
    cmds = decode_pie(sink / amp)
    queries = [b for k, b in cmds if k == "preamble"]
    acks = [b for k, b in cmds if k == "framesync"]
    rn16 = ["%04x" % int(b[2:], 2) for b in acks]
    json.dump({"amplitude": float(amp), "n_lead_cw": int(np.argmax(sink / amp < 0.5)),
               "queries": queries, "acks": acks, "rn16": rn16},
              open(os.path.join(HERE, "file_sink_commands.json"), "w"), indent=1)

    readme = open(os.path.join(REF, "README.md")).read().splitlines()
    open(os.path.join(HERE, "readme_expected.txt"), "w").write("\n".join(readme[45:53]) + "\n")

    from oracle.refflow import RefFlow
    iq = np.frombuffer(raw, dtype=np.complex64)
    for q, tag in ((0, "cfg1"), (4, "cfg1_q4")):
        r = RefFlow(q).run_stream(iq)
        np.save(os.path.join(HERE, tag + "_ref_records.npy"), r["records"])
        s = r["stats"]
        json.dump({"text": r["text"], "n_queries_sent": s.n_queries_sent,
                   "cur_inventory_round": s.cur_inventory_round, "cur_slot_number": s.cur_slot_number,
                   "n_epc_correct": s.n_epc_correct, "tag_reads": {str(k): v for k, v in s.tag_map().items()},
                   "n_windows": r["n_windows"]},
                  open(os.path.join(HERE, tag + "_ref_stats.json"), "w"), indent=1)
    reference_outputs(iq)
    rate_outputs()
    pulse_outputs()
    print("golden regenerated:", sorted(os.listdir(HERE)))


# inputs of the comparisons with the reference; the tests rebuild the same inputs
SYNTH_KW = [dict(n_tags=1), dict(n_tags=0), dict(n_tags=6, fixed_q=2), dict(n_tags=1, noise_sigma=0.02)]


def reader_script_bits():
    return np.random.default_rng(3).integers(0, 2, size=(9, 16)).astype(np.float32)


def tx_synth_rn16s():
    rn16s = np.random.default_rng(11).integers(0, 65536, size=12)
    rn16s[0], rn16s[1] = 0x0579, 0xFFFF     # first RN16 of the author's TX capture; all data-1
    return rn16s


def reference_outputs(iq):
    """oracle/_ref run on the inputs of the reference comparisons in tests/ -> reference_outputs.npz"""
    from gen2_uhf_rfid_reader_b200 import synth
    from oracle.refflow import RefFlow
    ref, ref4 = RefFlow(0), RefFlow(4)
    out = {}
    r = ref.run_stream(iq, want_tx=True)
    out["cfg1_tx"] = r["tx"]
    for chunk in (257, 4096, 100000):
        out["cfg1_records_chunk%d" % chunk] = ref.run_stream(iq, chunk=chunk)["records"]
    for i, kw in enumerate(SYNTH_KW):
        cap = synth.make_capture(48, seed=21, **kw)
        out["synth48_%d_records" % i], out["synth48_%d_counts" % i], _ = \
            ref.run_segments(cap["iq"].numpy(), cap["segments"], max_per_seg=4)
    cap = synth.make_capture(40, seed=5)
    out["synth40_records"], out["synth40_counts"], _ = ref.run_segments(cap["iq"].numpy(), cap["segments"], max_per_seg=4)
    out["reader_script_tx"], out["reader_script_nq"] = ref.reader_script(reader_script_bits())
    rn16s = tx_synth_rn16s()
    bits = ((rn16s[:, None] >> np.arange(15, -1, -1)[None, :]) & 1).astype(np.float32)
    for dac_rate in (1000000, 2000000):
        out["tx_synth_%d" % dac_rate], out["tx_synth_%d_nq" % dac_rate] = ref.reader_script(bits, dac_rate=dac_rate)
    out["tx_synth_q4"], _ = ref4.reader_script(np.zeros((2, 16), dtype=np.float32))
    np.savez_compressed(os.path.join(HERE, "reference_outputs.npz"), **out)


# (adc rate, taps) of the comparisons at other sample rates, one or more per kernel the library picks there:
# rx_fused_split_kernel<5,5> at 0.4 and 0.6 MS/s (n_T1 + 1 < 32: a gate opening fits inside one 32-sample mask word),
# rx_fused_split_kernel<5,0> / <5,5> at 1.0 MS/s, rx_pack_kernel at 1.2 MS/s, rx_fused_split_kernel<5,5> at 1.4-2.4 MS/s,
# rx_fused_kernel from 2.6 MS/s up.  Every one is a well-defined rate (tests/rate_rule.py).
RATES = [(400000, 25), (600000, 25), (1000000, 12), (1000000, 25), (1200000, 25), (1400000, 25), (1800000, 25),
         (2200000, 25), (2400000, 25), (2600000, 25), (3000000, 25), (5000000, 25), (4000000, 50), (8000000, 100)]
# capture variants: name -> make_capture keywords ("quiet": noise- and drift-free, which makes exact ties for the
# decoder's first-maximum rules)
RATE_VARIANTS = {"default": dict(), "quiet": dict(noise_sigma=0.0, clock_ppm_pct=0.0), "notag": dict(n_tags=0),
                 "noisy": dict(noise_sigma=0.02)}
RATE_Q4 = dict(fixed_q=4, n_tags=8)      # through the FIXED_Q = 4 build, at these rates only
RATE_Q4_RATES = (1200000, 2400000)
# heavy noise, at these rates only: rx_fused_kernel's rates have half_pw >= 3, where only noise dips of exactly half_pw
# samples test the gate's pulse-width rule at its boundary
RATE_GLITCH = dict(noise_sigma=0.2)
RATE_GLITCH_RATES = (2600000, 4000000)


def rate_cases():
    """(key, adc_rate, ntaps, make_capture keywords) of every stored comparison at other rates"""
    out = []
    for adc, ntaps in RATES:
        for name, kw in RATE_VARIANTS.items():
            out.append(("r%d_t%d_%s" % (adc, ntaps, name), adc, ntaps, kw))
        if adc in RATE_Q4_RATES:
            out.append(("r%d_t%d_q4" % (adc, ntaps), adc, ntaps, RATE_Q4))
        if adc in RATE_GLITCH_RATES:
            out.append(("r%d_t%d_glitch" % (adc, ntaps), adc, ntaps, RATE_GLITCH))
    return out


def rate_capture(adc, kw):
    from gen2_uhf_rfid_reader_b200 import synth
    return synth.make_capture(24, seed=31, adc_rate=adc, **kw)


def rate_outputs():
    """oracle/_ref on 24 segments at each rate and variant of rate_cases() -> reference_rates.npz"""
    from oracle.refflow import RefFlow
    ref = {0: RefFlow(0), 4: RefFlow(4)}
    out = {}
    for key, adc, ntaps, kw in rate_cases():
        cap = rate_capture(adc, kw)
        out[key + "_records"], out[key + "_counts"], _ = ref[kw.get("fixed_q", 0)].run_segments(
            cap["iq"].numpy(), cap["segments"], adc_rate=adc, ntaps=ntaps, max_per_seg=4)
    np.savez_compressed(os.path.join(HERE, "reference_rates.npz"), **out)


# Pulse-train captures (tests/test_gate_fsm.py): reader-like commands whose raw pulse widths, depths and quiet gaps are
# swept finely around n_PW and n_T1, so that after the boxcar the decimated pulse widths and gaps straddle the gate's
# bounds n_PW / 2 and n_T1.  One (adc rate, taps) per capture kernel configuration that decodes them.
PULSE_RATES = [(400000, 25), (1000000, 25), (1200000, 25), (2000000, 25), (2400000, 25), (2600000, 25),
               (4000000, 50), (8000000, 100)]
PULSE_MAX_WINDOWS = 8


def pulse_capture(adc, ntaps, n_segments=16, n_commands=8, decim=5):
    """raw I/Q (complex64 ndarray) and segments: per segment a carrier lead-in, then n_commands times: 6-8 low pulses
    (raw widths and depths swept around n_PW), a quiet gap swept around n_T1, one more pulse that ends the gap, and a
    stretch of carrier (the window) that sometimes ends before the window does"""
    from gen2_uhf_rfid_reader_b200 import abi
    from oracle.pyoracle import derive_cfg
    c = derive_cfg(adc_rate=adc, decim=decim, ntaps=ntaps)
    hp, t1 = c.n_PW // 2, c.n_T1
    rng = np.random.default_rng(adc // 1000 + ntaps)
    parts, offs, lens, off = [], [], [], 0
    for s in range(n_segments):
        amp = 0.8 * np.exp(1j * rng.uniform(0, 2 * np.pi))
        lvl = [np.ones(c.win_length * decim)]            # carrier lead-in: one avg_ampl window
        for k in range(n_commands):
            depth = rng.choice([0.0, 0.2, 0.4, 0.55])

            def pulse(sweep):
                # swept around n_PW / 2 after the boxcar, or clearly wider (a valid pulse)
                lo, hi = ((max(1, (hp - 3) * decim), (hp + 4) * decim + ntaps) if sweep else
                          ((hp + 2) * decim + ntaps // 2, (hp + 4) * decim + ntaps))
                lvl.append(np.full(rng.integers(lo, hi + 1), depth))

            for i in range(rng.integers(6, 9)):
                pulse(rng.random() < 0.3)
                lvl.append(np.ones(rng.integers(max(1, hp * decim), (3 * hp + 2) * decim + ntaps + 1)))
            lo, hi = (t1 - 1) * decim - ntaps // 2, (t1 + 2) * decim + ntaps // 2
            if rng.random() < 0.3:
                lo, hi = lo - 2 * decim - ntaps // 2, hi + 2 * decim + ntaps // 2
            lvl[-1] = np.ones(rng.integers(lo, hi + 1))   # the quiet gap
            pulse(False)
            lvl.append(np.ones(rng.integers(c.len_rn16, c.len_epc + 200) * decim))
        x = np.concatenate(lvl) * amp
        x = x + (rng.standard_normal(x.size) + 1j * rng.standard_normal(x.size)) * 0.004
        parts.append(x.astype(np.complex64))
        offs.append(off)
        lens.append(x.size)
        off += x.size
    return np.concatenate(parts), abi.make_segments(offs, lens)


def pulse_outputs():
    """oracle/_ref on the pulse-train capture of each PULSE_RATES entry -> reference_pulses.npz"""
    from oracle.refflow import RefFlow
    ref = RefFlow(0)
    out = {}
    for adc, ntaps in PULSE_RATES:
        iq, segs = pulse_capture(adc, ntaps)
        key = "p%d_t%d" % (adc, ntaps)
        out[key + "_records"], out[key + "_counts"], _ = ref.run_segments(iq, segs, adc_rate=adc, ntaps=ntaps,
                                                                          max_per_seg=PULSE_MAX_WINDOWS)
    np.savez_compressed(os.path.join(HERE, "reference_pulses.npz"), **out)


if __name__ == "__main__":
    if sys.argv[1:] == ["rates"]:
        rate_outputs()
    elif sys.argv[1:] == ["pulses"]:
        pulse_outputs()
    else:
        main()
