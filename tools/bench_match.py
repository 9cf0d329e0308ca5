"""Cost and yield of the EPC match (rfid_b200_match_epc) next to the capture decode, on one GPU.

At cfg4 size (160,000 simulated 2 MS/s slots, Q = 4, 8 tags, open loop, 2 windows per slot), at the simulator's default
tag gain and at 0.004, for dictionaries of K = 8 (the tags' frames), 1,024 and 65,536 (the tags' frames and random ones):
  * the match call and decode_capture, CUDA events per call, the arms alternating round by round (median and min);
  * the prepare and score kernels apart, from torch.profiler's CUDA activity in a run of their own;
  * the score kernel's achieved int8 rate 2 N K 128 / kernel time (N attempted windows) against the 1,979 TOPS dense
    data-sheet figure of the H100 SXM;
  * reads: CRC passes, recoveries, MATCHED windows, and MATCHED windows that name a frame other than the simulator's
    truth for the slot (or lie in an empty slot).
Prints the card's name and power limit read in the same run, and one JSON line per gain and K.
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

PEAK_INT8_TOPS = 1979.0


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def timed(arms, rounds):
    for f in arms.values():
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


def kernel_times(f, reps=5):
    """mean device time per call of each rx_match_* kernel, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    f()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("prepare", "score", "init"):
            if "rx_match_%s_kernel" % name in ev.key:
                out[name] = round(ev.device_time_total / reps, 1) if hasattr(ev, "device_time_total") else \
                    round(ev.cuda_time_total / reps, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nseg", type=int, default=160000)
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    print("card:", card())
    rx = capi.Gen2Rx(fixed_q=4)
    nseg, mw = args.nseg, 2
    default_gain = capi.default_sim().tag_gain
    for g in (default_gain, 0.004):
        cap = rx.sim_capture(capi.default_sim(n_tags=8, closed_loop=0, seed=5, tag_gain=g), nseg)
        iq, segs = cap["iq"], cap["segs"]
        truth = cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1)
        tap, res, cnt = rx._decode_tapped(iq, segs, mw, capi.SC16_SCALE)
        qual = rx.window_quality(tap, res, cnt, mw)
        fix = rx.recover_epc(tap, res, cnt, qual, mw)
        recs, _ = capi.results_to_numpy(res, cnt, mw)
        fx, _ = capi.fixes_to_numpy(fix, cnt, mw)
        frames = np.unique(truth["epc"][truth["n_replies"] > 0], axis=0)
        rng = np.random.default_rng(12)
        res2, cnt2 = torch.empty_like(res), torch.empty_like(cnt)
        for K in (8, 1024, 65536):
            extra = synth.make_epc_frames(rng.integers(0, 256, (max(0, K - frames.shape[0]), 12)).astype(np.uint8))
            d = torch.from_numpy(np.concatenate([frames, extra])[:K].copy()).cuda()
            match = torch.empty((nseg * mw, 32), dtype=torch.uint8, device="cuda")
            mc = torch.empty((K, 16), dtype=torch.uint8, device="cuda")

            def run():
                rx.match_epc(tap, res, cnt, d, mw, fixes=fix, match=match, match_count=mc)
            arms = {"decode": lambda: rx.decode_capture(iq, segs, max_windows=mw, results=res2, counts=cnt2),
                    "match": run}
            out = {"tag_gain": g, "nseg": nseg, "K": K, "rounds": args.rounds, **timed(arms, args.rounds)}
            kt = kernel_times(run)
            m, _ = capi.matches_to_numpy(match, cnt, mw)
            st = m[:, 1]["status"]
            n_rows = int(((st == abi.MATCH_MATCHED) | (st == abi.MATCH_AMBIGUOUS) | (st == abi.MATCH_NO_MATCH)).sum())
            matched = st == abi.MATCH_MATCHED
            dn = d.cpu().numpy()
            wrong = matched & ((truth["n_replies"] == 0) | (dn[np.maximum(m[:, 1]["entry"], 0)] != truth["epc"]).any(1))
            out.update({"kernel_us": kt, "rows": n_rows,
                        "score_int8_tops": round(2.0 * n_rows * K * 128 / (kt["score"] * 1e-6) / 1e12, 1)
                        if kt.get("score") else None,
                        "crc_ok": int((recs[:, 1]["crc_ok"] == 1).sum()),
                        "recovered": int((fx[:, 1]["status"] == abi.FIX_RECOVERED).sum()),
                        "matched": int(matched.sum()), "ambiguous": int((st == abi.MATCH_AMBIGUOUS).sum()),
                        "wrong_matched": int(wrong.sum()),
                        "empty_slots_matched": int((matched & (truth["n_replies"] == 0)).sum())})
            if out["score_int8_tops"] is not None:
                out["score_of_datasheet_int8"] = round(out["score_int8_tops"] / PEAK_INT8_TOPS, 3)
            print(json.dumps(out), flush=True)
            del match, mc, d
        del iq, tap, res, cnt, qual, fix, res2, cnt2, cap
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
