"""Cost and yield of EPC recovery (rfid_b200_recover_epc) next to the capture decode, on one GPU.

At cfg4 size (160,000 simulated 2 MS/s slots, Q = 4, 8 tags) and at two tag gains (the simulator's default and a weak
0.004) it times, with CUDA events, four arms on the same capture, alternating them round by round: decode_capture alone,
decode with the window tap set, the quality kernel on that tap, and the recovery kernel on the tap and the quality
records.  It counts the windows attempted and recovered, the EPC reads before and after recovery, and the recovered
EPCs that differ from the simulator's truth (there must be none).  Prints the card's name and power limit read in the
same run, and one JSON line per gain.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen2_uhf_rfid_reader_b200 import abi, capi  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nseg", type=int, default=160000)
    ap.add_argument("--gains", default="default,0.004")
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    print("card:", card())
    rx = capi.Gen2Rx(fixed_q=4)
    nseg, mw = args.nseg, 2
    for gain in args.gains.split(","):
        kw = {} if gain == "default" else dict(tag_gain=float(gain))
        sim = capi.default_sim(n_tags=8, closed_loop=0, seed=5, **kw)
        cap = rx.sim_capture(sim, nseg)
        iq, segs = cap["iq"], cap["segs"]
        tap = torch.empty(nseg * mw * rx.len_epc, dtype=torch.complex64, device="cuda")
        res = torch.zeros((nseg * mw, 64), dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        qual = torch.zeros((nseg * mw, 16), dtype=torch.uint8, device="cuda")
        fix = torch.zeros((nseg * mw, 32), dtype=torch.uint8, device="cuda")

        def decode(with_tap):
            rx.set_window_tap(tap if with_tap else None)
            rx.decode_capture(iq, segs, max_windows=mw, results=res, counts=cnt)
            rx.set_window_tap(None)

        arms = {"decode": lambda: decode(False), "decode_tap": lambda: decode(True),
                "quality": lambda: rx.window_quality(tap, res, cnt, mw, quality=qual),
                "recover": lambda: rx.recover_epc(tap, res, cnt, qual, mw, fixes=fix)}
        times = {k: [] for k in arms}
        for f in arms.values():   # warm-up, in the order the arms depend on each other
            f()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for k, f in arms.items():
                e0.record()
                f()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3)
        recs, counts = capi.results_to_numpy(res, cnt, mw)
        fx, _ = capi.fixes_to_numpy(fix, cnt, mw)
        truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
        st = fx[:, 1]["status"]
        rec = st == abi.FIX_RECOVERED
        wrong = rec & (fx[:, 1]["bits"] != truth["epc"]).any(axis=1)
        q, _ = capi.quality_to_numpy(qual, cnt, mw)
        before = int((recs[:, 1]["crc_ok"] == 1).sum())
        after = int((capi.apply_fixes(recs, counts, fx)[:, 1]["crc_ok"] == 1).sum())
        out = {"nseg": nseg, "tag_gain": sim.tag_gain, "rounds": args.rounds,
               "median_us": {k: float(np.median(v)) for k, v in times.items()},
               "min_us": {k: float(np.min(v)) for k, v in times.items()},
               "attempted": int(((st >= abi.FIX_RECOVERED) & (st <= abi.FIX_FAILED)).sum()),
               "recovered": int(rec.sum()), "ambiguous": int((st == abi.FIX_AMBIGUOUS).sum()),
               "epc_reads_before": before, "epc_reads_after": after,
               "wrong_recoveries": int(wrong.sum()),
               "wrong_snr_db": [round(float(10 * np.log10(v)), 2) for v in q[wrong, 1]["snr"]],
               "wrong_n_flips": fx[wrong, 1]["n_flips"].tolist(), "wrong_n_replies": truth["n_replies"][wrong].tolist()}
        print(json.dumps(out))
        del tap, res, cnt, qual, fix, cap, iq, segs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
