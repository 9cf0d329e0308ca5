"""Developer measurement: reader-command decoding (Gen2Rx.decode_commands) against the capture decode on one GPU.

  python tools/bench_commands.py [--runs 5] [--steps 20] [--cfg3-steps 3] [--out DIR]

Workloads from the library's CUDA slot simulator, as tools/bench_sc16.py builds them: cfg2 (1000 slots x 16,960 raw
samples) and cfg3 (100,000 slots), each as an sc16 capture and its fc32 conversion.  Per workload and run, alternating
the arms: CUDA-event time of `steps` back-to-back calls of decode_commands and of decode_capture on the same capture, in
both formats.  Bytes/s at 8 B (fc32) or 4 B (sc16) per sample and their share of the 3.35 TB/s data-sheet HBM bandwidth
follow from the time per call.  Checks: sc16 commands equal fc32 commands bit for bit, and every slot opens with a Query
or QueryRep and carries the ACK the simulator sent.  Prints the card's name, power limit and maximum SM clock.
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_sc16 import HBM_BPS, card, make_workload  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="calls per timed run at cfg2")
    ap.add_argument("--cfg3-steps", type=int, default=3, help="calls per timed run at cfg3")
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()

    import torch
    from gen2_uhf_rfid_reader_b200 import abi, capi
    assert torch.cuda.is_available(), "bench_commands.py needs a GPU"
    scale = capi.SC16_SCALE
    out = {"card": card(), "workloads": {}}
    print("card (name, power limit, max SM clock):", out["card"], flush=True)
    rx = capi.Gen2Rx()
    stream = torch.cuda.current_stream()
    MW, MC = 2, 4
    ok = True
    for name, nslots, steps in (("cfg2", 1000, args.steps), ("cfg3", 100000, args.cfg3_steps)):
        q, x, segs, truth = make_workload(rx, nslots, scale)
        n_raw = q.shape[0]
        nseg = segs.numel() // 16
        res = torch.zeros((nseg * MW, 64), dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        cmd = torch.zeros((nseg * MC, 64), dtype=torch.uint8, device="cuda")
        ccnt = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        rx.decode_commands(q, segs, MC, cmd, ccnt, stream, scale=scale)
        c16 = capi.commands_to_numpy(cmd.clone(), ccnt.clone(), MC)
        rx.decode_commands(x, segs, MC, cmd, ccnt, stream)
        c32 = capi.commands_to_numpy(cmd.clone(), ccnt.clone(), MC)
        same = c16[0].tobytes() == c32[0].tobytes() and c16[1].tolist() == c32[1].tolist()
        cmds, counts = c32
        acked = truth["acked_rn16"] >= 0
        first = cmds[:, 0]
        truth_ok = bool((counts == 1 + acked).all()
                        and (first["kind"] == np.where(truth["is_query"] == 1, abi.TX_QUERY, abi.TX_QUERY_REP)).all()
                        and (cmds[acked, 1]["arg"] == truth["acked_rn16"][acked]).all())
        ok = ok and same and truth_ok
        arms = {
            "commands_fc32": lambda: rx.decode_commands(x, segs, MC, cmd, ccnt, stream),
            "commands_sc16": lambda: rx.decode_commands(q, segs, MC, cmd, ccnt, stream, scale=scale),
            "capture_fc32": lambda: rx.decode_capture(x, segs, MW, res, cnt, stream),
            "capture_sc16": lambda: rx.decode_capture(q, segs, MW, res, cnt, stream, scale=scale),
        }
        times = {a: [] for a in arms}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for run in range(args.runs):
            for a in (list(arms) if run % 2 == 0 else list(arms)[::-1]):
                arms[a]()   # warm
                e0.record(stream)
                for _ in range(steps):
                    arms[a]()
                e1.record(stream)
                e1.synchronize()
                times[a].append(e0.elapsed_time(e1) / steps)
        rows = {}
        for a, ts in times.items():
            t = float(np.median(ts)) * 1e-3
            b = 4 if a.endswith("sc16") else 8
            rows[a] = {"ms_per_call": [round(v, 4) for v in ts], "ms_median": t * 1e3, "gb_per_s": b * n_raw / t / 1e9,
                       "hbm_fraction": b * n_raw / t / HBM_BPS}
        w = {"slots": nslots, "raw_samples": n_raw, "sc16_equals_fc32": same, "commands_equal_truth": truth_ok,
             "arms": rows}
        out["workloads"][name] = w
        print(name, json.dumps(w), flush=True)
        del q, x, res, cnt, cmd, ccnt
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_commands.json"), "w") as f:
            json.dump(out, f, indent=1)
    print("checks:", "ok" if ok else "FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
