"""Cost of the window-quality pass (rfid_b200_window_quality) next to the capture decode, on one GPU.

At cfg2 (1,000 segments) and cfg4 (160,000 segments, Q = 4, 8 tags) sizes of simulated 2 MS/s slots it times, with CUDA
events, four arms on the same capture, alternating them round by round: decode_capture alone, decode with the window tap
set (one extra write of every stored window), the quality kernel alone on that tap, and decode with the tap followed by
the quality kernel.  Prints the card's name and power limit read in the same run, and one JSON line per size.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen2_uhf_rfid_reader_b200 import capi  # noqa: E402

SIZES = {"cfg2": dict(nseg=1000, fixed_q=0, n_tags=1), "cfg4": dict(nseg=160000, fixed_q=4, n_tags=8)}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="cfg2,cfg4")
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    print("card:", card())
    for name in args.sizes.split(","):
        cfg = SIZES[name]
        rx = capi.Gen2Rx(fixed_q=cfg["fixed_q"])
        sim = capi.default_sim(n_tags=cfg["n_tags"], closed_loop=0, seed=5)
        cap = rx.sim_capture(sim, cfg["nseg"])
        iq, segs, mw, nseg = cap["iq"], cap["segs"], 2, cfg["nseg"]
        tap = torch.empty(nseg * mw * rx.len_epc, dtype=torch.complex64, device="cuda")
        res = torch.zeros((nseg * mw, 64), dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        qual = torch.zeros((nseg * mw, 16), dtype=torch.uint8, device="cuda")

        def decode(with_tap):
            rx.set_window_tap(tap if with_tap else None)
            rx.decode_capture(iq, segs, max_windows=mw, results=res, counts=cnt)
            rx.set_window_tap(None)

        arms = {"decode": lambda: decode(False), "decode_tap": lambda: decode(True),
                "quality": lambda: rx.window_quality(tap, res, cnt, mw, quality=qual),
                "decode_tap_quality": lambda: (decode(True), rx.window_quality(tap, res, cnt, mw, quality=qual))}
        times = {k: [] for k in arms}
        for f in arms.values():   # warm-up
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
        q, c = capi.quality_to_numpy(qual, cnt, mw)
        recs, _ = capi.results_to_numpy(res, cnt, mw)
        out = {"size": name, "nseg": nseg, "tap_bytes": tap.numel() * 8,
               "median_us": {k: float(np.median(v)) for k, v in times.items()},
               "min_us": {k: float(np.min(v)) for k, v in times.items()},
               "summary": capi.inventory_summary(recs, c, q)}
        print(json.dumps(out))
        del tap, rx


if __name__ == "__main__":
    main()
