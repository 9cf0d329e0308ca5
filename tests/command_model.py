"""numpy restatement of the reader-command decoder (include/rfid_b200.h, csrc/rx_cmd.cuh) -- test infrastructure.

One segment at a time, independent of everything outside it:
  p = re*re + im*im (float32, three roundings); thr2 = (level_frac*level_frac) * max p, or level_abs*level_abs;
  low = p < thr2; a fall is a low sample whose predecessor in the segment is high (a low first sample is one);
  a burst starts at a fall with no low sample before it or whose previous low sample is >= gap samples back;
  bursts of >= 4 falls are PIE commands: tari = d0, rtcal = d1, preamble iff d2 > rtcal (trcal = d2), every further
  fall-to-fall interval d is one bit, 1 iff 2*d > rtcal.
"""
import numpy as np

from gen2_uhf_rfid_reader_b200 import abi, synth

CMD_OTHER = -1
COMMAND_DTYPE = abi.COMMAND_DTYPE


def gap_samples(gap_us, adc_rate):
    return int(float(np.float32(gap_us)) * 1e-6 * adc_rate)


def _classify(sync_pre, bits):
    """(kind, arg, crc_ok) of a command's data bits (list of 0/1)"""
    n = len(bits)
    s = "".join(str(b) for b in bits)
    val = lambda a, b: int(s[a:b], 2)  # noqa: E731
    if sync_pre:
        if n == 22 and s.startswith("1000"):
            crc = synth.crc5_gen2(bits[:17])
            return abi.TX_QUERY, val(13, 17), int(crc == list(bits[17:]))
        return CMD_OTHER, -1, -1
    if n == 4 and s.startswith("00"):
        return abi.TX_QUERY_REP, val(2, 4), -1
    if n == 18 and s.startswith("01"):
        return abi.TX_ACK, val(2, 18), -1
    if n == 9 and s.startswith("1001"):
        return abi.TX_QUERY_ADJUST, val(4, 6), -1
    if n == 8 and s == "11000000":
        return abi.TX_NAK, -1, -1
    return CMD_OTHER, -1, -1


def decode_segment(x, adc_rate=2_000_000, level_frac=0.5, level_abs=0.0, gap_us=400.0, segment=0):
    """complex64 samples of one segment -> COMMAND_DTYPE records (all of them, in order)"""
    x = np.ascontiguousarray(x, dtype=np.complex64)
    re, im = x.real.astype(np.float32), x.imag.astype(np.float32)
    p = re * re + im * im
    if level_abs > 0:
        thr2 = np.float32(level_abs) * np.float32(level_abs)
    else:
        peak = np.max(p, initial=np.float32(0), where=~np.isnan(p))   # NaN samples never win (nor are they low)
        thr2 = (np.float32(level_frac) * np.float32(level_frac)) * peak
    low = p < thr2
    prev = np.concatenate(([False], low[:-1]))
    falls = np.flatnonzero(low & ~prev)
    lows = np.flatnonzero(low)
    gap = gap_samples(gap_us, adc_rate)
    k = np.searchsorted(lows, falls, side="left") - 1
    prev_low = np.where(k >= 0, lows[np.maximum(k, 0)], -1)
    starts = np.flatnonzero((prev_low < 0) | (falls - prev_low - 1 >= gap))
    out = []
    for b, i0 in enumerate(starts):
        i1 = starts[b + 1] if b + 1 < starts.size else falls.size
        f = falls[i0:i1]
        if f.size < 4:
            continue
        last_low = prev_low[i1] if i1 < falls.size else lows[-1]
        d = np.diff(f)
        tari, rtcal = int(d[0]), int(d[1])
        pre = int(d[2]) > rtcal
        trcal = int(d[2]) if pre else 0
        bits = [int(2 * int(v) > rtcal) for v in d[(3 if pre else 2):]]
        kind, arg, crc = _classify(pre, bits)
        r = np.zeros((), dtype=COMMAND_DTYPE)
        r["segment"], r["index"] = segment, len(out)
        r["start"], r["end"] = int(f[0]), int(last_low) + 1
        r["kind"], r["n_bits"] = kind, len(bits)
        r["tari"], r["rtcal"], r["trcal"] = tari, rtcal, trcal
        r["crc_ok"], r["arg"] = crc, arg
        packed = np.packbits(np.array(bits[:128] + [0] * (128 - min(128, len(bits))), dtype=np.uint8))
        r["bits"] = packed
        out.append(r)
    return np.array(out, dtype=COMMAND_DTYPE)


def decode_segments(iq, segs, max_commands, **kw):
    """the device call's layout: (records [nseg, max_commands], counts [nseg])"""
    iq = np.asarray(iq)
    nseg = len(segs)
    recs = np.zeros((nseg, max_commands), dtype=COMMAND_DTYPE)
    counts = np.zeros(nseg, dtype=np.int32)
    for s in range(nseg):
        o, n = int(segs[s]["offset"]), int(segs[s]["length"])
        r = decode_segment(iq[o:o + n], segment=s, **kw)
        counts[s] = r.size
        k = min(r.size, max_commands)
        recs[s, :k] = r[:k]
    return recs, counts


def bits_str(rec):
    n = min(int(rec["n_bits"]), 128)
    return "".join(str(b) for b in np.unpackbits(rec["bits"])[:n])
