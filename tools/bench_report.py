"""Cost of the tag inventory report (rfid_b200_tag_report) next to the capture decode, on one GPU, and what its power
and phase numbers mean.

Timing (CUDA events per call, the arms alternating round by round, median and min):
  * cfg4 size: 160,000 simulated 2 MS/s slots (Q = 4, 8 tags, open loop), 2 windows per slot: decode_capture alone, the
    report on the records and quality records, and on the records, quality and fix records;
  * two adversarial tables of 320,000 stored slots that are all reads: of one EPC, and of 320,000 distinct EPCs.
Calibration: make_capture(600, seed=77) (one tag, known per-slot gain g and phase) decoded with recovery; for every read
it compares |h| / ntaps with |g| and arg h with arg g, and the report's peak_rssi_db with 20 log10 of the largest |g|
among the tag's reads.  Prints the card's name and power limit read in the same run, and one JSON line per part.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen2_uhf_rfid_reader_b200 import abi, capi, synth  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def timed(arms, rounds):
    for f in arms.values():   # warm-up, in the order the arms depend on each other
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, f in arms.items():
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e3)
    return {"median_us": {k: round(float(np.median(v)), 1) for k, v in times.items()},
            "min_us": {k: round(float(np.min(v)), 1) for k, v in times.items()}}


def adversarial(distinct, nseg=160000, seed=11):
    rng = np.random.default_rng(seed)
    recs = np.zeros(nseg * 2, dtype=abi.RESULT_DTYPE)
    recs["kind"], recs["crc_ok"] = abi.EPC, 1
    bits = np.zeros((recs.size, 16), dtype=np.uint8)
    bits[:, 0] = 0x30
    if distinct:
        bits[:, 2:10] = rng.permutation(recs.size).astype(">u8").view(np.uint8).reshape(-1, 8)
        bits[:, 10:16] = rng.integers(0, 256, (recs.size, 6))
    recs["bits"] = bits
    recs["h_re"], recs["h_im"] = rng.standard_normal((2, recs.size)).astype(np.float32)
    segs = abi.make_segments(np.arange(nseg, dtype=np.uint64) * 16960, np.full(nseg, 16960))
    return (torch.from_numpy(recs.view(np.uint8).copy()).cuda(), torch.full((nseg,), 2, dtype=torch.int32, device="cuda"),
            capi.segments_to_device(segs, "cuda"))


def calibrate(rx, n=600, seed=77, gains=(0.0227, 0.004)):
    out = []
    for g in gains:
        cap = synth.make_capture(n, device="cuda", seed=seed, tag_gain=g)
        segs = capi.segments_to_device(cap["segments"], "cuda")
        res, cnt, _, _, tags, summary, rt = rx.decode_capture_report(cap["iq"], segs, 2)
        recs, _ = capi.results_to_numpy(res, cnt, 2)
        t, _ = capi.tags_to_numpy(tags, summary)
        read = rt.cpu().numpy().reshape(-1, 2)[:, 1] >= 0
        # the simulator's per-slot gain of its one tag (synth.make_capture: one round per slot at Q = 0)
        amp, ph = np.zeros(n), np.zeros(n)
        for i in range(n):
            r = np.random.Generator(np.random.Philox(key=[seed, i]))
            r.integers(0, 1, size=1)
            amp[i] = g * r.uniform(0.6, 1.4, size=1)[0]
            ph[i] = synth.TAG_DIR + r.uniform(-0.6, 0.6, size=1)[0]
        h = recs[:, 1]["h_re"].astype(np.float64) + 1j * recs[:, 1]["h_im"].astype(np.float64)
        ratio = np.abs(h[read]) / rx.params.ntaps / amp[read]
        dphi = np.degrees(np.angle(h[read] * np.exp(-1j * ph[read])))
        row = capi.tag_table(t, ntaps=rx.params.ntaps)[0]
        out.append({"tag_gain": g, "reads": int(read.sum()),
                    "abs_h_over_ntaps_gain": [round(float(np.percentile(ratio, p)), 4) for p in (5, 50, 95)],
                    "arg_h_minus_arg_g_deg": [round(float(np.percentile(dphi, p)), 2) for p in (5, 50, 95)],
                    "peak_rssi_db": round(float(row["peak_rssi_db"]), 2),
                    "20log10_max_gain_db": round(float(20 * np.log10(amp[read].max())), 2),
                    "last_phase_deg": round(float(row["last_phase_deg"]), 2)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nseg", type=int, default=160000)
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    print("card:", card())
    rx = capi.Gen2Rx(fixed_q=4)
    nseg, mw = args.nseg, 2
    cap = rx.sim_capture(capi.default_sim(n_tags=8, closed_loop=0, seed=5), nseg)
    iq, segs = cap["iq"], cap["segs"]
    res, cnt, qual, fix = rx.decode_capture_recover(iq, segs, max_windows=mw)
    rt = torch.empty(nseg * mw, dtype=torch.int32, device="cuda")
    tb = torch.empty((1024, 64), dtype=torch.uint8, device="cuda")
    sb = torch.empty(32, dtype=torch.uint8, device="cuda")
    res2 = torch.empty_like(res)
    cnt2 = torch.empty_like(cnt)
    kw = dict(tags=tb, summary=sb, read_tag=rt)
    arms = {"decode": lambda: rx.decode_capture(iq, segs, max_windows=mw, results=res2, counts=cnt2),
            "report_quality": lambda: rx.tag_report(res, cnt, segs, mw, quality=qual, **kw),
            "report_quality_fixes": lambda: rx.tag_report(res, cnt, segs, mw, quality=qual, fixes=fix, **kw)}
    out = {"workload": "cfg4", "nseg": nseg, "rounds": args.rounds, **timed(arms, args.rounds)}
    tags, summary, _ = rx.tag_report(res, cnt, segs, mw, quality=qual, fixes=fix)
    t, sm = capi.tags_to_numpy(tags, summary)
    out.update({"n_tags": int(sm["n_tags"]), "reads": int(sm["reads"]), "recovered": int(sm["recovered"]),
                "rejected_length": int(sm["rejected_length"]), "rejected_empty": int(sm["rejected_empty"]),
                "input_mb": round(nseg * mw * (64 + 16 + 32) / 1e6, 1)})
    print(json.dumps(out))
    del iq, res2, cnt2, res, cnt, qual, fix, cap
    torch.cuda.empty_cache()
    tb = torch.empty((400000, 64), dtype=torch.uint8, device="cuda")
    sb = torch.empty(32, dtype=torch.uint8, device="cuda")
    for distinct in (False, True):
        r, c, s = adversarial(distinct)
        rt = torch.empty(r.shape[0], dtype=torch.int32, device="cuda")
        arms = {"report": lambda: rx.tag_report(r, c, s, 2, max_tags=400000, tags=tb, summary=sb, read_tag=rt)}
        res = timed(arms, args.rounds)
        sm = capi.tags_to_numpy(tb, sb)[1]
        print(json.dumps({"workload": "distinct EPCs" if distinct else "one EPC", "slots": int(r.shape[0]) // 64,
                          "n_tags": int(sm["n_tags"]), **res}))
    for row in calibrate(capi.Gen2Rx()):
        print(json.dumps({"calibration": row}))


if __name__ == "__main__":
    main()
