"""Calibration of rfid_b200_match_epc's defaults on the CPU (numpy restatement tests/match_model.py, the oracle's windows).

Costs are printed in mean reliabilities (D / 16).  Parts, every one seeded:
  noise      best-of-K D1 of 10^5 Gaussian windows (r_j ~ N(0, 1), seed 91) against K = 16 / 1,024 / 65,536 random frames
             (seed 92), and of the EPC windows of the 612 empty slots of make_capture(1024, seed=78, fixed_q=4,
             n_tags=8, tag_gain=0.004);
  replies    D1 of every failing EPC window against its true frame, make_capture(600, seed=77) at tag_gain 0.004 /
             0.003 / 0.0025 (one tag), and the MATCHED / AMBIGUOUS / NO_MATCH counts at the defaults with the truth
             plus 1,023 random frames as the dictionary;
  held-out   the same windows with the true frame removed: against 1,024 random frames, and against dictionaries of one
             CRC-valid decoy at sign distance 4..16 from it (PC length field intact, four per distance, seed 93) plus
             1,023 random frames: how often the decoy is MATCHED (or AMBIGUOUS), by distance.
Prints one JSON line per part.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import match_model as mm  # noqa: E402
import quality_model as qm  # noqa: E402
import recover_model as rm  # noqa: E402
from gen2_uhf_rfid_reader_b200 import synth  # noqa: E402


def random_frames(k, seed):
    rng = np.random.default_rng(seed)
    return synth.make_epc_frames(rng.integers(0, 256, size=(k, 12)).astype(np.uint8))


def best_d1(q, s, frames, ks, chunk=1024):
    """smallest cost over the first k frames, for every k in ks: {k: D1 [N]} (float32 products are exact here: every
    partial sum is an integer below 2^24)"""
    cw = torch.from_numpy(mm.codeword_signs(frames).astype(np.float32))
    out = {k: np.zeros(q.shape[0], dtype=np.int64) for k in ks}
    for i in range(0, q.shape[0], chunk):
        qq = torch.from_numpy(q[i:i + chunk].astype(np.float32))
        ss = torch.from_numpy(s[i:i + chunk].astype(np.float32))
        D = (qq * ss).sum(1, keepdim=True) + (qq * (1 - 2 * ss)) @ cw.T
        for k in ks:
            out[k][i:i + chunk] = D[:, :k].min(1).values.round().long().numpy()
    return out


def pct(x):
    x = np.asarray(x, dtype=np.float64) / 16.0
    return [round(float(v), 2) for v in (x.min(), np.percentile(x, 1), np.median(x), x.max())] if x.size else []


def failing_projections(oracle, cap):
    w, r, c = qm.oracle_windows(oracle, cap["iq"].numpy(), cap["segments"], 2)
    n_f, len_epc = oracle.cfg.n_tag_bit_f, oracle.cfg.len_epc
    fail = np.nonzero(r[:, 1]["crc_ok"] == 0)[0]
    rr = np.stack([rm.epc_projections(w[s, 1], r[s, 1], n_f, len_epc) for s in fail]) if fail.size else \
        np.zeros((0, 128), np.float32)
    return fail, rr, r, c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--noise", type=int, default=100_000)
    args = ap.parse_args()
    from oracle.pyoracle import Oracle
    oracle = Oracle()
    ks = (16, 1024, 65536)
    frames = random_frames(65536, 92)
    # noise
    r = np.random.default_rng(91).standard_normal((args.noise, 128)).astype(np.float32)
    q, s, _ = mm.reliabilities(r)
    b = best_d1(q, s, frames, ks)
    print(json.dumps({"part": "gaussian", "n": args.noise, **{"K=%d" % k: pct(b[k]) for k in ks},
                      **{"K=%d_below_%d" % (k, t): int((b[k] <= 16 * t).sum()) for k in ks for t in (12, 16, 20)}}))
    cap = synth.make_capture(1024, device="cpu", seed=78, fixed_q=4, n_tags=8, tag_gain=0.004)
    w, rec, c = qm.oracle_windows(oracle, cap["iq"].numpy(), cap["segments"], 2)
    empty = np.nonzero(cap["truth"]["n_replies"] == 0)[0]
    re = np.stack([rm.epc_projections(w[i, 1], rec[i, 1], oracle.cfg.n_tag_bit_f, oracle.cfg.len_epc) for i in empty])
    q, s, _ = mm.reliabilities(re)
    b = best_d1(q, s, frames, ks)
    print(json.dumps({"part": "empty slots", "n": int(empty.size), **{"K=%d" % k: pct(b[k]) for k in ks}}))
    # replies and held-out tags
    rng = np.random.default_rng(93)
    for g in (0.004, 0.003, 0.0025):
        cap = synth.make_capture(600, device="cpu", seed=77, tag_gain=g)
        fail, rr, recs, _ = failing_projections(oracle, cap)
        truth = cap["truth"]["epc"][fail]
        q, s, _ = mm.reliabilities(rr)
        own = mm.costs(q, s, mm.codeword_signs(truth))[np.arange(fail.size), np.arange(fail.size)] if fail.size else []
        others = random_frames(1023, 94)
        d = mm.match_projections(rr, np.concatenate([truth[:1], others]))
        st = np.bincount(d["status"], minlength=6)
        wrong = int(((d["status"] == mm.MATCHED) & (d["entry"] != 0)).sum())
        held = mm.match_projections(rr, random_frames(1024, 95))
        dec, dist = mm.decoys(truth[0], 13 * 4, rng)   # four decoys at each sign distance 4..16
        held_rand = random_frames(1023, 96)
        hit = np.zeros(17, dtype=np.int64)
        amb = np.zeros(17, dtype=np.int64)
        for f, w in zip(dec, dist):   # one decoy in a dictionary of 1,024
            hd = mm.match_projections(rr, np.concatenate([f[None], held_rand]))
            hit[w] += int(((hd["status"] == mm.MATCHED) & (hd["entry"] == 0)).sum())
            amb[w] += int(((hd["status"] == mm.AMBIGUOUS) & (hd["entry"] == 0)).sum())
        print(json.dumps({"part": "replies", "tag_gain": g, "read": int((recs[:, 1]["crc_ok"] == 1).sum()),
                          "failing": int(fail.size), "own_cost": pct(own),
                          "own_cost_le": {t: int((np.asarray(own) <= 16 * t).sum()) for t in (8, 12, 16, 20)},
                          "matched": int(st[mm.MATCHED]), "ambiguous": int(st[mm.AMBIGUOUS]),
                          "no_match": int(st[mm.NO_MATCH]), "wrong": wrong,
                          "held_out_random_matched": int((held["status"] == mm.MATCHED).sum()),
                          "decoy_trials": int(fail.size * dec.shape[0]), "decoy_matched": int(hit.sum()),
                          "decoy_matched_by_distance_4_16": hit[4:].tolist(),
                          "decoy_ambiguous_by_distance_4_16": amb[4:].tolist()}))


if __name__ == "__main__":
    main()
