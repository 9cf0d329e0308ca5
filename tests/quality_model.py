"""numpy restatement of the window-quality rule (include/rfid_b200.h, csrc/rx_quality.cuh) -- test infrastructure.

Per stored window, from its DC-removed samples w[0, length) and its record (sync_index, h, T, length):
  projections  r_j = Re((s_a - s_b) * conj(h)) at the decoder's own sample positions, in float32 with every operation
               rounded: RN16 the 32 half-bits jm = index + half + ... + half, k = round(jm); EPC the 128 pairs
               a = (int)(j*(2T) + index), b = (int)(2j*T + T + index) (samples outside the window are 0);
  snr          m = S1/k, (m*m) / (S2/k - m*m), S1 = sum |r_j|, S2 = sum r_j^2 in float64; +inf for a zero denominator;
  energy       mean |w|^2 over the reply [sync_index, e) / mean |w|^2 over the noise reference [0, sync_index - 2n/5)
               and [e, length) (n = n_tag_bit_i), |w|^2 = re^2 + im^2 in float64; e = the decoder's position two
               half-bits after its last decision sample (RN16 round(jm_33), EPC b_128) + n/5; when the reference holds
               fewer than n samples its tail is moved back to make up n;
every sum lane-strided (term i to lane i % 32, ascending) and then over the 32 lane sums in ascending lane order; both
ratios rounded once to float32.  Outcome: EMPTY unless energy >= empty_ratio; an RN16 window is then SINGLE if
snr >= single_ratio, else COLLISION; an EPC window is SINGLE.
"""
import numpy as np

import rate_rule

f32, f64 = np.float32, np.float64

EMPTY, SINGLE, COLLISION = 0, 1, 2
QUALITY_DTYPE = np.dtype([("energy", "<f4"), ("snr", "<f4"), ("outcome", "<i4"), ("n_decisions", "<i4")])
DEFAULT_EMPTY_DB = 9.5
DEFAULT_SINGLE_SNR_DB = 8.8


def ratios(empty_db=DEFAULT_EMPTY_DB, single_snr_db=DEFAULT_SINGLE_SNR_DB):
    """the host's linear thresholds: 10^(dB/10) in double of the float settings"""
    return 10.0 ** (float(f32(empty_db)) / 10.0), 10.0 ** (float(f32(single_snr_db)) / 10.0)


def canonical(v):
    """float64 -> float32 rounded once, every NaN as 0x7fc00000 (the kernel's one NaN pattern)"""
    return f32(np.nan) if np.isnan(v) else f32(v)


def lane_sum(terms):
    """float64 terms -> their sum in the kernel's order (lane-strided partial sums, then lanes ascending)"""
    t = np.asarray(terms, dtype=f64).ravel()
    t = np.concatenate([t, np.zeros((-t.size) % 32)])
    part = np.zeros(32)
    for row in t.reshape(-1, 32):
        part = part + row
    total = 0.0
    for v in part:
        total += float(v)
    return total


def _proj(sa, sb, h):
    x = (sa.real - sb.real).astype(f32)
    y = (sa.imag - sb.imag).astype(f32)
    return (x * f32(h.real)).astype(f32) - (y * f32(-h.imag)).astype(f32)


def data_index(sync_index, n_f):
    """first data sample, sync index + 6.5 symbols, as the decoder rounds it"""
    half = f32(n_f * f32(0.5))
    return int(f32(f32(f32(sync_index) + f32(f32(6.0) * n_f)) + half))


def positions(kind, sync_index, T, n_f, n_i):
    """decoder sample positions: (a, b) index arrays of the k projections and the reply's end (the decoder's position
    two half-bits after its last decision sample, plus n_i // 5); for an RN16 window also the float half-bit positions
    jm (the decoder's have-test)"""
    index = data_index(sync_index, n_f)
    half = f32(n_f * f32(0.5))
    if kind == 0:
        jm = np.zeros(34, dtype=f32)
        jm[0] = f32(index)
        for m in range(33):
            jm[m + 1] = f32(jm[m] + half)
        k = np.floor(jm.astype(f64) + 0.5).astype(np.int64)    # roundf: halves away from zero (jm >= 0)
        return k[0:32:2], k[1:32:2], int(k[33]) + n_i // 5, jm[:32]
    T = f32(T)
    two_t = f32(f32(2.0) * T)
    j = np.arange(129)
    a = (f32(j.astype(f32) * two_t) + f32(index)).astype(f32).astype(np.int64)
    b = (f32(f32(f32((2 * j).astype(f32) * T) + T)) + f32(index)).astype(f32).astype(np.int64)
    return a[:128], b[:128], int(b[128]) + n_i // 5, None


def projections(w, n, a, b, h):
    """r_j of sample pairs (a_j, b_j) of window w[0, n) (w has one extra element, 0, for samples outside the window)"""
    take = lambda p: w[np.where((p >= 0) & (p < n), p, n)]    # noqa: E731
    return _proj(take(a), take(b), h)


def decisions(w, rec, n_f):
    """the projections of a window (length n = record length) and the bits the decoder makes of their signs (FM0:
    a bit is 1 where the sign differs from the previous one, which starts positive)"""
    n = int(rec["length"])
    w = np.concatenate([np.ascontiguousarray(w[:n], dtype=np.complex64), np.zeros(1, dtype=np.complex64)])
    h = np.complex64(complex(f32(rec["h_re"]), f32(rec["h_im"])))
    a, b, _, _ = positions(int(rec["kind"]), int(rec["sync_index"]), rec["T"], f32(n_f), 0)
    r = projections(w, n, a, b, h)
    pos = r > 0
    bits = pos != np.concatenate([[True], pos[:-1]])
    return r, np.packbits(bits.astype(np.uint8))


def spans(sync_index, reply_end, n, n_i, lead=None):
    """(reply, head, tail) half-open sample ranges.  The noise reference is the head [0, sync_index - lead), before the
    reply and the matched filter's delay of it, and the tail [reply_end, n) after it; when the two hold fewer than n_i
    samples, the tail is moved back to make up n_i (into the reply's end)."""
    lead = 2 * n_i // 5 if lead is None else lead
    h1 = min(max(sync_index - lead, 0), n)
    t0 = min(reply_end, n)
    if h1 + (n - t0) < n_i:
        t0 = max(n - (n_i - h1), h1)
    return (sync_index, min(reply_end, t0)), (0, h1), (t0, n)


def window_quality(w, rec, n_f, n_i, len_epc, empty_ratio, single_ratio, lead=None):
    """one quality record (QUALITY_DTYPE scalar) of window samples w (complex64) and its RESULT_DTYPE record"""
    out = np.zeros((), dtype=QUALITY_DTYPE)
    kind = int(rec["kind"])
    n = max(0, min(int(rec["length"]), len_epc))
    w = np.concatenate([np.ascontiguousarray(w[:n], dtype=np.complex64), np.zeros(1, dtype=np.complex64)])
    h = np.complex64(complex(f32(rec["h_re"]), f32(rec["h_im"])))
    sync = int(rec["sync_index"])
    a, b, reply_end, jm = positions(kind, sync, rec["T"], f32(n_f), n_i)
    if kind == 0 and not (jm < f32(n)).all():
        out["energy"] = out["snr"] = np.nan
        out["outcome"], out["n_decisions"] = EMPTY, 0
        return out
    r = projections(w, n, a, b, h)
    k = r.size
    r64 = r.astype(f64)
    m = lane_sum(np.abs(r64)) / k
    s2 = lane_sum(r64 * r64) / k
    num = m * m
    den = s2 - num
    with np.errstate(divide="ignore", invalid="ignore"):
        out["snr"] = np.inf if den == 0.0 else canonical(f64(num) / den)
    p2 = w.real.astype(f64) ** 2 + w.imag.astype(f64) ** 2
    (r0, r1), (h0, h1), (t0, t1) = spans(sync, reply_end, n, n_i, lead)
    noise = np.concatenate([p2[h0:h1], p2[t0:t1]])
    if r0 < 0 or r1 <= r0 or noise.size == 0:
        out["energy"] = np.nan
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            out["energy"] = canonical((f64(lane_sum(p2[r0:r1])) / (r1 - r0)) / (f64(lane_sum(noise)) / noise.size))
    out["n_decisions"] = k
    e, s = float(out["energy"]), float(out["snr"])
    if not e >= empty_ratio:
        out["outcome"] = EMPTY
    elif kind != 0 or s >= single_ratio:
        out["outcome"] = SINGLE
    else:
        out["outcome"] = COLLISION
    return out


def quality(windows, recs, counts, adc_rate=2_000_000, empty_db=DEFAULT_EMPTY_DB, single_snr_db=DEFAULT_SINGLE_SNR_DB,
            decim=5, lead=None):
    """the device call's layout: windows [nseg, max_windows, len_epc] complex64, recs RESULT_DTYPE [nseg, max_windows]
    -> QUALITY_DTYPE [nseg, max_windows], zero beyond the stored records"""
    n_i, n_f, _, len_epc = derived(adc_rate, decim)
    er, sr = ratios(empty_db, single_snr_db)
    nseg, mw = recs.shape
    out = np.zeros((nseg, mw), dtype=QUALITY_DTYPE)
    for s in range(nseg):
        for k in range(min(max(int(counts[s]), 0), mw)):
            out[s, k] = window_quality(windows[s, k], recs[s, k], n_f, n_i, len_epc, er, sr, lead)
    return out


def oracle_windows(oracle, iq, segs, max_windows):
    """the oracle's gate windows and decoded records per segment, in the window tap's layout:
    (windows complex64 [nseg, max_windows, len_epc], recs RESULT_DTYPE [nseg, max_windows], counts int32 [nseg])"""
    from gen2_uhf_rfid_reader_b200 import abi
    L = oracle.cfg.len_epc
    nseg = len(segs)
    wins = np.zeros((nseg, max_windows, L), dtype=np.complex64)
    recs = np.zeros((nseg, max_windows), dtype=abi.RESULT_DTYPE)
    counts = np.zeros(nseg, dtype=np.int32)
    for s in range(nseg):
        o, n = int(segs[s]["offset"]), int(segs[s]["length"])
        g = oracle.gate(oracle.mf(iq[o:o + n]), want_windows=True)
        counts[s] = g["n"]
        for k in range(min(g["n"], max_windows)):
            kind = k & 1
            length = oracle.cfg.len_epc if kind else oracle.cfg.len_rn16
            wins[s, k, :length] = g["windows"][k, :length]
            r = oracle.decode_window(kind, wins[s, k, :length])
            r["segment"], r["window"], r["open_index"] = s, k, g["open_idx"][k]
            recs[s, k] = r
    return wins, recs, counts


def early_windows(oracle, iq, d):
    """the gate windows of one continuous capture, each opened d decimated samples early (the reply sits d samples later
    in its window, as for a tag with a longer T1), with their DC estimates, and the oracle's records of them:
    (windows complex64 [1, n, len_epc], recs RESULT_DTYPE [1, n], counts [1])"""
    from gen2_uhf_rfid_reader_b200 import abi
    y = oracle.mf(iq)
    g = oracle.gate(y)
    m = g["n"]
    L = oracle.cfg.len_epc
    wins = np.zeros((1, m, L), dtype=np.complex64)
    recs = np.zeros((1, m), dtype=abi.RESULT_DTYPE)
    for k in range(m):
        kind = k & 1
        length = L if kind else oracle.cfg.len_rn16
        o = int(g["open_idx"][k]) - d
        wins[0, k, :length] = y[o:o + length] - g["dc"][k]
        r = oracle.decode_window(kind, wins[0, k, :length])
        r["window"], r["open_index"] = k, o
        recs[0, k] = r
    return wins, recs, np.array([m], dtype=np.int32)


def derived(adc_rate, decim=5):
    """(n_tag_bit_i, n_tag_bit_f, len_rn16, len_epc) of a rate, as the library derives them"""
    n_i, n_f, l_rn16, l_epc = rate_rule.derived(np.array([adc_rate]), decim)
    return int(n_i[0]), f32(n_f[0]), int(l_rn16[0]), int(l_epc[0])


def noise_extents(adc_rate, decim=5):
    """over every sync index the preamble search can return and, for EPC windows, every candidate half-period T:
    ((RN16, EPC) fewest reply samples, fewest noise-reference samples, fewest noise-reference samples that lie outside
    [sync_index - lead, reply_end), i.e. before or after the reply)"""
    n_i, n_f, len_rn16, len_epc = derived(adc_rate, decim)
    sync_range = int(np.ceil(1.5 * float(n_f)))
    n64 = float(n_f)
    lo, hi = f32(n64 / 2.0 - n64 / 2.0 / 100), f32(n64 / 2.0 + n64 / 2.0 / 100)
    steps = [f32(lo + f32(f32(f32(t) * f32(hi - lo)) / f32(19))) for t in range(20)]
    reply, noise, clean = [], [], []
    for kind, n, Ts in ((0, len_rn16, [f32(0)]), (1, len_epc, steps)):
        r, no, cl = [], [], []
        for s in range(sync_range):
            for T in Ts:
                e = positions(kind, s, T, n_f, n_i)[2]
                (r0, r1), (h0, h1), (t0, t1) = spans(s, e, n, n_i)
                r.append(r1 - r0)
                no.append((h1 - h0) + (t1 - t0))
                cl.append((h1 - h0) + (t1 - max(t0, e)) if t1 > max(t0, e) else (h1 - h0))
        reply.append(min(r))
        noise.append(min(no))
        clean.append(min(cl))
    return tuple(reply), tuple(noise), tuple(clean)
