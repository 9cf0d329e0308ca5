#!/usr/bin/env python
"""Developer aid: build the library with RFID_B200_PHASE_PROFILE and print the timeline (cycles since CTA start) of the
pack kernel's warps A / B / C of segment 0 and of the chain warp of CTA 0, the decode phases of segment 0's windows, and
per CTA its lifetime and the time from its last window closing at a gate to its last decode done (GPU box).  RFID_B200_LIB selects an already
built profiling library instead; RFID_B200_PACK_G forces the segments per CTA (as in the library)."""
import os, sys, subprocess
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gen2_uhf_rfid_reader_b200 import build
PACK_MAX_SEG = 8   # kPMaxSeg (csrc/rx_pack.cuh)
lib = os.environ.get("RFID_B200_LIB") or os.path.join(ROOT, "gen2_uhf_rfid_reader_b200", "librfid_b200_prof.so")
if not os.path.exists(lib) or os.environ.get("REBUILD"):
    subprocess.check_call(["nvcc"] + build.NVCC_FLAGS + ["-DRFID_B200_PHASE_PROFILE", "-o", lib, os.path.join(build.CSRC, "rfid_b200.cu")])
os.environ["RFID_B200_LIB"] = lib
import gen2_uhf_rfid_reader_b200.capi as capi
from gen2_uhf_rfid_reader_b200 import synth
dev = torch.device("cuda:0")
nseg = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
rx = capi.Gen2Rx()
cap = synth.make_capture(nseg, seed=3, device=dev)
segs = capi.segments_to_device(cap["segments"], dev)
tap = torch.zeros((nseg * 2, rx.len_epc), dtype=torch.complex64, device=dev)
for it in range(3):
    rx.decode_capture(cap["iq"], segs, 2)
torch.cuda.synchronize()
rx.set_window_tap(tap)
rx.decode_capture(cap["iq"], segs, 2)
torch.cuda.synchronize()
raw_log = tap.view(torch.int64).cpu().numpy().reshape(-1)
log = raw_log[: 320 * 8].reshape(320, 8)
# segments per CTA as the library picks them (pack_segments_per_cta): enough to fill every SM once, at most PACK_MAX_SEG
sms = torch.cuda.get_device_properties(dev).multi_processor_count
G = int(os.environ.get("RFID_B200_PACK_G", "0")) or min(PACK_MAX_SEG, max(1, -(-nseg // sms)))
ncta = (nseg + G - 1) // G
print("G = %d segments per CTA, %d CTAs on %d SMs" % (G, ncta, sms))
ct = raw_log[512 * 8: 512 * 8 + 4 * ncta].reshape(ncta, 4)[:, :3].astype(np.float64)
t0 = ct[:, 0].min()
st, en, cl = (ct[:, 0] - t0) / 1000.0, (ct[:, 1] - t0) / 1000.0, (ct[:, 2] - t0) / 1000.0
life, tail = en - st, en - cl
pct = lambda v: "min %.2f p50 %.2f p90 %.2f max %.2f" % (v.min(), np.percentile(v, 50), np.percentile(v, 90), v.max())
print("CTAs %d: start us min %.2f max %.2f | last decode done us: %s | CTA 0: %.2f .. %.2f" % (ncta, st.min(), st.max(), pct(en), st[0], en[0]))
print("CTA lifetime us: %s" % pct(life))
print("last window closed by a gate -> last decode done, us: %s" % pct(tail))
order = np.argsort(en)
print("slowest CTAs:", [(int(i), round(float(en[i]), 2)) for i in order[-6:]], "fastest:", [(int(i), round(float(en[i]), 2)) for i in order[:4]])
A, B, CH, C = log[0:64], log[64:128], log[128:192], log[192:256]
steps = 14 + 2
print("B sub-phases: tile | avg ready  pre-masks  masks  fsm  rebuild  P3done")
for i in range(steps):
    print("%3d | %7d %7d %7d %7d %7d %7d" % (i, B[i][1], B[i][4], B[i][5], B[i][6], B[i][7], B[i][2]))
print("tile | A0: start blocksums |y|stored P1end | A1: start P1end | B: start avg-ready P3done | chain: start inputs-ready done")
A1 = log[256:320] if log.shape[0] >= 320 else A
for i in range(steps):
    print("%3d | %7d %7d %7d %7d | %7d %7d | %7d %7d %7d | %7d %7d %7d" %
          (i, A[i][0], A[i][1], A[i][2], A[i][3], A1[i][0], A1[i][3], B[i][0], B[i][1], B[i][2], CH[i][0], CH[i][1], CH[i][2]))
for k in range(2):
    print("window %d: opened seen %d, first phase %d, finish starts %d, decoded %d" % (k, C[k][0], C[k][1], C[k][3], C[k][2]))
e = C[60]
print("EPC decode of segment 0 (cycles of work): head+sync %d, period search %d in %d chunks before the finish + %d in it, "
      "bit samples %d, bits+crc %d; finish %d" % (e[1] - e[0], e[5], e[7], e[2] - e[6], e[3] - e[2], e[4] - e[3], e[4] - e[6]))
r = C[61]
print("RN16 decode of segment 0 (cycles): head+sync %d, bit decisions %d, total %d" % (r[1] - r[0], r[4] - r[6], r[4] - r[0]))
nclaim = int(raw_log[1023 * 8])
if nclaim:
    cl = raw_log[1024 * 8: 1024 * 8 + 4 * min(nclaim, 1024)].reshape(-1, 4)
    what = {1: "head", 2: "chunk", 3: "rest"}
    print("decoder claims of CTA 0 (%d), by pool warp (C0.., then A1 of segment id - D): segment/window what@phase start-end" % nclaim)
    for d in sorted(set(int(c[0]) & 0xff for c in cl)):
        rows = sorted((c for c in cl if int(c[0]) & 0xff == d), key=lambda c: c[1])
        busy = sum(int(c[2] - c[1]) for c in rows)
        print("  C%d busy %d:" % (d, busy), " ".join("%d/%d %s@%d %d-%d" % ((int(c[0]) >> 8) & 0xff, (int(c[0]) >> 16) & 0xff,
              what.get((int(c[0]) >> 24) & 0xf, "?"), (int(c[0]) >> 28) & 0xf, c[1], c[2]) for c in rows))
