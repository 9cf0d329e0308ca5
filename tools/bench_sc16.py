"""Developer measurement: complex int16 (sc16) captures against float32 (fc32) ones on one GPU.

  python tools/bench_sc16.py [--runs 5] [--steps 20] [--cfg3-steps 3] [--parent-lib PATH] [--out DIR]

Workloads from the library's CUDA slot simulator (Gen2Rx.sim_capture): cfg2 (1000 slots x 16,960 raw samples) and cfg3
(100,000 slots).  Each capture is quantised on the GPU, q = round(x / scale) clamped to int16, and its fc32 partner is
q.float() * scale.  Per workload and run, alternating the arms: kernel time (CUDA events, rfid_b200_kernel_time) of
`steps` decodes of the sc16 capture, of its fc32 partner, and -- with --parent-lib, a librfid_b200.so built from another
commit -- of the fc32 partner through that library.  Raw GSamples/s, bytes/s at 4 B (sc16) or 8 B (fc32) per sample and
their share of the 3.35 TB/s data-sheet HBM bandwidth follow from the kernel time.  Then end-to-end ingest
(ingest_capture_host on a pinned host recording from synth.make_capture, wall clock per call) in both formats, and the
throughput of the two exact int16 -> float forms (tests/cuda/sc16_harness.cu).  Checks: sc16 records equal fc32 records
bit for bit, and the decisions equal the simulator's truth.  Prints the card's name, power limit and maximum SM clock.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12     # H100 SXM data sheet


class ParentRx:
    """the fc32 capture path of another build of librfid_b200.so (raw ctypes: it need not have the sc16 entry points)"""

    def __init__(self, path):
        from gen2_uhf_rfid_reader_b200 import abi, capi
        self.lib = L = C.CDLL(path)
        vp = C.c_void_p
        L.rfid_b200_create.argtypes = [C.POINTER(abi.Params), C.POINTER(vp)]
        L.rfid_b200_decode_capture.argtypes = [vp, vp, C.c_size_t, vp, C.c_int, C.c_int, vp, vp, vp]
        L.rfid_b200_enable_kernel_timing.argtypes = [vp, C.c_int]
        L.rfid_b200_kernel_time.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]
        self.h = vp()
        assert L.rfid_b200_create(C.byref(capi.default_params()), C.byref(self.h)) == 0

    def decode_capture(self, iq, segs, max_windows, results, counts, stream):
        nseg = segs.numel() // 16
        assert self.lib.rfid_b200_decode_capture(self.h, iq.data_ptr(), iq.numel(), segs.data_ptr(), nseg, max_windows,
                                                 results.data_ptr(), counts.data_ptr(), stream.cuda_stream) == 0

    def enable_kernel_timing(self, on=True):
        self.lib.rfid_b200_enable_kernel_timing(self.h, int(on))

    def kernel_time(self, reset=True):
        ms, n = C.c_float(0), C.c_int(0)
        self.lib.rfid_b200_kernel_time(self.h, int(reset), C.byref(ms), C.byref(n))
        return ms.value, n.value


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def make_workload(rx, nslots, scale, chunk=10000):
    """simulated slots -> (q int16 [n, 2] CUDA, x complex64 CUDA = its conversion, segs CUDA, truth ndarray)"""
    import torch
    from gen2_uhf_rfid_reader_b200 import abi, capi
    sim = capi.default_sim()
    seg_len = rx.sim_segment_length(sim)
    n = nslots * seg_len
    q = torch.empty((n, 2), dtype=torch.int16, device="cuda")
    segs, truth = [], []
    for first in range(0, nslots, chunk):
        k = min(chunk, nslots - first)
        cap = rx.sim_capture(sim, k, first_segment=first)
        q[first * seg_len:(first + k) * seg_len] = torch.round(torch.view_as_real(cap["iq"]) / scale).clamp(-32768, 32767).to(torch.int16)
        s = cap["segs"].cpu().numpy().view(abi.SEGMENT_DTYPE).reshape(-1).copy()
        s["offset"] += first * seg_len
        segs.append(s)
        truth.append(cap["truth"].cpu().numpy().view(abi.SIM_TRUTH_DTYPE).reshape(-1))
        del cap
    x = torch.view_as_complex((q.float() * scale).contiguous())
    segs = np.concatenate(segs)
    return q, x, capi.segments_to_device(segs, "cuda"), np.concatenate(truth)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="decodes per timed run at cfg2")
    ap.add_argument("--cfg3-steps", type=int, default=3, help="decodes per timed run at cfg3")
    ap.add_argument("--parent-lib", default=None, help="another build of librfid_b200.so: its fc32 path joins the A/B")
    ap.add_argument("--ingest-rounds", type=int, default=4000)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()

    import torch
    from gen2_uhf_rfid_reader_b200 import abi, capi, synth
    from gen2_uhf_rfid_reader_b200.build import SC16_HARNESS, SC16_HARNESS_SRC, build_harness
    assert torch.cuda.is_available(), "bench_sc16.py needs a GPU"
    scale = capi.SC16_SCALE
    out = {"card": card(), "scale": scale, "workloads": {}}
    print("card (name, power limit, max SM clock):", out["card"], flush=True)
    rx = capi.Gen2Rx()
    parent = ParentRx(args.parent_lib) if args.parent_lib else None
    stream = torch.cuda.current_stream()
    MW = 2

    for name, nslots, steps in (("cfg2", 1000, args.steps), ("cfg3", 100000, args.cfg3_steps)):
        q, x, segs, truth = make_workload(rx, nslots, scale)
        n_raw = q.shape[0]
        nseg = segs.numel() // 16
        res = torch.zeros((nseg * MW, 64), dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        # checks: sc16 = fc32 bit for bit, decisions = truth
        rx.decode_capture(q, segs, MW, res, cnt, stream, scale=scale)
        torch.cuda.synchronize()
        r16, c16 = capi.results_to_numpy(res.clone(), cnt.clone(), MW)
        rx.decode_capture(x, segs, MW, res, cnt, stream)
        torch.cuda.synchronize()
        r32, c32 = capi.results_to_numpy(res.clone(), cnt.clone(), MW)
        same = r16.tobytes() == r32.tobytes() and c16.tolist() == c32.tolist()
        truth_ok = bool((c16 == 2).all() and (r16[:, 0]["tag_id"] == truth["strongest_rn16"]).all()
                        and (r16[:, 1]["crc_ok"] == 1).all() and (r16[:, 1]["bits"] == truth["epc"]).all())
        if parent is not None:
            parent.decode_capture(x, segs, MW, res, cnt, stream)
            torch.cuda.synchronize()
            rp, cp = capi.results_to_numpy(res.clone(), cnt.clone(), MW)
            parent_same = rp.tobytes() == r32.tobytes() and cp.tolist() == c32.tolist()
        arms = {"sc16": (rx, q, dict(scale=scale)), "fc32": (rx, x, {})}
        if parent is not None:
            arms["fc32_parent"] = (parent, x, {})
        times = {a: [] for a in arms}
        for run in range(args.runs):
            order = list(arms) if run % 2 == 0 else list(arms)[::-1]
            for a in order:
                r, iq, kw = arms[a]
                r.decode_capture(iq, segs, MW, res, cnt, stream, **kw)   # warm
                torch.cuda.synchronize()
                r.enable_kernel_timing(True)
                r.kernel_time(reset=True)
                for _ in range(steps):
                    r.decode_capture(iq, segs, MW, res, cnt, stream, **kw)
                torch.cuda.synchronize()
                ms, k = r.kernel_time(reset=True)
                r.enable_kernel_timing(False)
                times[a].append(ms / k)
        rows = {}
        for a, ts in times.items():
            t = float(np.median(ts)) * 1e-3
            b = 4 if a == "sc16" else 8
            rows[a] = {"kernel_ms": [round(v, 4) for v in ts], "kernel_ms_median": t * 1e3, "gsamples_per_s": n_raw / t / 1e9,
                       "bytes_per_sample": b, "gb_per_s": b * n_raw / t / 1e9, "hbm_fraction": b * n_raw / t / HBM_BPS}
        w = {"slots": nslots, "raw_samples": n_raw, "sc16_equals_fc32": same, "decisions_equal_truth": truth_ok, "arms": rows}
        if parent is not None:
            w["parent_equals_fc32"] = parent_same
        out["workloads"][name] = w
        print(name, json.dumps(w), flush=True)
        del q, x, res, cnt
        torch.cuda.empty_cache()

    # end-to-end ingest from pinned host memory, both formats, alternating
    cap = synth.make_capture(args.ingest_rounds, seed=1234, device="cuda")
    qd = torch.round(torch.view_as_real(cap["iq"]) / scale).clamp(-32768, 32767).to(torch.int16)
    hq = torch.empty(qd.shape, dtype=torch.int16).pin_memory()
    hq.copy_(qd)
    hx = torch.empty(qd.shape[0], dtype=torch.complex64).pin_memory()
    hx.copy_(torch.view_as_complex(qd.float() * scale))
    srcs = {"sc16": hq.numpy().ravel(), "fc32": hx.numpy()}
    ing = {a: [] for a in srcs}
    got = {}
    for a, s in srcs.items():
        got[a] = rx.ingest_capture_host(s, max_windows=4)
    ing_same = all(got["sc16"][k].tobytes() == got["fc32"][k].tobytes() for k in range(3))
    for run in range(args.runs):
        for a in (list(srcs) if run % 2 == 0 else list(srcs)[::-1]):
            t0 = time.perf_counter()
            rx.ingest_capture_host(srcs[a], max_windows=4)
            ing[a].append(time.perf_counter() - t0)
    n_raw = qd.shape[0]
    out["ingest"] = {"rounds": args.ingest_rounds, "raw_samples": n_raw, "sc16_equals_fc32": ing_same,
                     "segments": int(len(got["sc16"][0])),
                     "arms": {a: {"seconds_per_call": [round(v, 5) for v in ts], "median_s": float(np.median(ts)),
                                  "gsamples_per_s": n_raw / float(np.median(ts)) / 1e9} for a, ts in ing.items()}}
    print("ingest", json.dumps(out["ingest"]), flush=True)

    # the two exact int16 -> float forms (throughput)
    h = C.CDLL(build_harness(SC16_HARNESS_SRC, SC16_HARNESS))
    h.sc16_harness_rate.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_float)]
    blocks = 132 * 16
    sink = torch.empty(blocks * 256, dtype=torch.float32, device="cuda")
    forms = {}
    for form, label in ((0, "i2f"), (1, "iadd_fadd")):
        ms = C.c_float(0)
        assert h.sc16_harness_rate(form, blocks, 4096, 6, sink.data_ptr(), C.byref(ms)) == 0
        forms[label] = {"ms": ms.value, "gconversions_per_s": 2.0 * blocks * 256 * 4096 / (ms.value * 1e-3) / 1e9}
    out["conversion_forms"] = forms
    print("conversion", json.dumps(forms), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sc16.json"), "w") as f:
            json.dump(out, f, indent=1)
    ok = all(w["sc16_equals_fc32"] and w["decisions_equal_truth"] and w.get("parent_equals_fc32", True)
             for w in out["workloads"].values()) and ing_same
    print("checks:", "ok" if ok else "FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
