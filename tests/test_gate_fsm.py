"""The gate's threshold masks and closed-run state machine (csrc/rx_gate.cuh: gate_masks<W>, gate_closed_run<W>) against
a per-sample replay of the reference gate (gate_impl.cc:136-180).

gate_closed_run is a bit-parallel rewrite of the reference's sample loop; every capture kernel decides with it where a
window opens.  Here it runs alone, one warp per case (tests/cuda/gate_harness.cu), on about half a million single-tile cases
per tile width W and on a few thousand 64-tile streams, at every (n_T1, n_PW / 2) of a defined configuration and at the
corners of the function's precondition, and every result is compared exactly with `replay`: the reference's loop,
sample by sample, vectorised over the cases.  The replay also labels each case by the rule of the rewrite that decided
it, and the tests assert that every rule was reached.

The replay itself is pinned to the restatement's gate (Oracle.gate) on the recording, on the captures at every
sample rate of the rate comparisons and on the pulse-train captures (CPU).

The single-tile count is a trade-off: the numpy case generator and replay, not the GPU, take the time, and 2 x 2^18
cases per W keep the module near one minute.  Rules that random cases reach rarely get their own generators (pulse
trains aimed at the opening position) and a minimum count each, which matters more than the total.

The pulse-train captures (make_golden.pulse_capture) test what the harness cannot: the gate logic at the call sites of
every capture kernel, decoded end to end against the reference's blocks.
"""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden import PULSE_MAX_WINDOWS, PULSE_RATES, RATE_VARIANTS, RATES, pulse_capture, rate_capture  # noqa: E402
from rate_rule import GRID, well_defined  # noqa: E402

NUM_PULSES_COMMAND = 5          # global_vars.h: more valid pulses than this make a reader command
THRESH_FRACTION = np.float32(0.75)
NEITHER, BELOW, ABOVE = 0, 1, 2  # a sample vs. its threshold


# ------------------------------------------------------------------ the reference's loop, sample by sample
def replay(sym, run_from, nvalid, n_T1, half_pw, sig_pos, n_samples, num_pulses, windows=None, max_open=64,
           tile=None, labels=True):
    """gate_impl.cc:145-180 on symbols sym [positions, cases] (NEITHER / BELOW / ABOVE), every case at once.

    Samples [run_from, nvalid) of each case are closed samples.  Without `windows` the run ends at its first opening
    (one closed run, what gate_closed_run computes).  With windows = (first length, second length) the gate stays open
    after an opening by the reference's ungate rule (n_samples counts to n_samples_to_ungate; GATE_SEEK_* then sets
    n_samples to 0; window lengths alternate) and the closed samples after it go on (a stream of tiles of `tile`
    samples).

    Returns ret (first opening or -1), opens [cases, max_open] and n_open, the final sig_pos, n_samples, num_pulses and
    gate_open, and the labels of the rules that decided (_LABELS)."""
    P, N = sym.shape
    pos = np.asarray(sig_pos, bool).copy()
    ns = np.asarray(n_samples, np.int64).copy()
    npl = np.asarray(num_pulses, np.int64).copy()
    n_T1, half_pw = np.asarray(n_T1, np.int64), np.asarray(half_pw, np.int64)
    run_from, nvalid = np.asarray(run_from, np.int64), np.asarray(nvalid, np.int64)
    np0 = npl.copy()
    gate_open = np.zeros(N, bool)
    live = np.ones(N, bool)               # one closed run: not opened yet
    opens = np.full((N, max_open), -1, np.int64)
    n_open = np.zeros(N, np.int64)
    rows = np.arange(N)
    if windows is not None:
        to_ungate = np.asarray(windows[0], np.int64).copy()
        wcount = np.zeros(N, np.int64)
        close_tile = np.full(N, -1, np.int64)
    L = {k: np.zeros(N, bool) for k in _LABELS}
    n_edges = np.zeros(N, np.int64)       # edges of the run up to the opening
    open_edges = np.full(N, -1, np.int64)
    valid_rises = np.zeros(N, np.int64)
    invalid_seen = np.zeros(N, bool)
    epos = pos.copy()                     # signal_state over the whole run (an opening leaves it as it is)
    e_first = np.full(N, -1, np.int64)
    edge_word = np.zeros(((P + 31) // 32, N), bool)
    for p in range(P):
        act = (p >= run_from) & (p < nvalid)
        s = sym[p]
        b, a = s == BELOW, s == ABOVE
        closed = act & ~gate_open & live
        if labels and windows is None:
            # the edges of the whole run
            ef, er = act & epos & b, act & ~epos & a
            epos = (epos & ~ef) | er
            edge_word[p >> 5] |= ef | er
            e_first = np.where((e_first < 0) & (ef | er), p, e_first)
        # ---- gate_impl.cc:145-162
        ns = ns + (act & live)                                   # :145 (and :184 while open)
        fall = closed & pos & b                                  # :148
        rise = closed & ~pos & a                                 # :154
        valid = rise & (ns > half_pw)                            # :157
        if labels:
            eq = s == NEITHER
            L["fall_at_open"] |= fall & (ns > n_T1) & (npl > NUM_PULSES_COMMAND)
            L["equal_high"] |= closed & pos & eq
            L["equal_low"] |= closed & ~pos & eq
            first = rise & (n_edges == 0)
            L["first_rise_invalid"] |= first & ~valid
            L["first_rise_at_half_pw"] |= first & (ns == half_pw)
            L["pulse_half_pw"] |= rise & (n_edges > 0) & (ns == half_pw)
            L["pulse_half_pw_1"] |= rise & (n_edges > 0) & (ns == half_pw + 1)
            invalid_seen |= rise & ~valid
            valid_rises += valid
            n_edges += fall | rise
        pos = (pos & ~fall) | rise
        npl = np.where(rise, np.where(valid, npl + 1, 0), npl)   # :157-160
        ns = np.where(fall | rise, 0, ns)                        # :150, :161
        # ---- :164-179
        op = closed & pos & (ns > n_T1) & (npl > NUM_PULSES_COMMAND)
        if op.any():
            if labels:
                L["carried_pulses_open"] |= op & ~invalid_seen & (np0 > 0) & (valid_rises > 0) & \
                    (npl - np0 <= NUM_PULSES_COMMAND)
                open_edges = np.where(op & (open_edges < 0), n_edges, open_edges)
                if windows is not None:
                    L["reopen_in_tile"] |= op & (close_tile == p // tile)
            k = op & (n_open < max_open)
            opens[rows[k], n_open[k]] = p
            n_open += op
            npl = np.where(op, 0, npl)
            ns = np.where(op, 1, ns)
            if windows is None:
                live &= ~op
        if windows is not None:
            # ---- :182-195 (the trigger sample is the window's first)
            shut = act & gate_open & (ns >= to_ungate)
            gate_open = (gate_open & ~shut) | op
            if shut.any():
                wcount += shut
                to_ungate = np.where(shut, np.where(wcount & 1, windows[1], windows[0]), to_ungate)
                ns = np.where(shut, 0, ns)                       # GATE_SEEK_* (:112-123)
                if labels:
                    close_tile = np.where(shut, p // tile, close_tile)
                    valid_rises = np.where(shut, 0, valid_rises)
    ret = np.where(n_open > 0, opens[:, 0], -1)
    if labels and windows is None:
        _labels(L, sym, ret, open_edges, e_first, edge_word, run_from, nvalid, n_T1, sig_pos, n_samples, num_pulses,
                invalid_seen, valid_rises)
    return dict(ret=ret, opens=opens, n_open=n_open, sig_pos=pos, n_samples=ns, num_pulses=npl, gate_open=gate_open,
                labels=L)


# the rules of gate_closed_run, as labels of the cases that reach them
_LABELS = ["carrier", "carrier_open", "carried_open", "carried_open_on_edge", "short_open", "long_open",
           "long_open_no_free_word", "word_skip", "first_rise_invalid", "first_rise_at_half_pw", "pulse_half_pw",
           "pulse_half_pw_1", "fall_at_open", "open_at_last", "carried_pulses_open", "carried_pulses_final",
           "equal_high", "equal_low", "reopen_in_tile"]


def _labels(L, sym, ret, open_edges, e_first, edge_word, run_from, nvalid, n_T1, sig_pos, n_samples, num_pulses,
            invalid_seen, valid_rises):
    opened = ret >= 0
    sig_pos = np.asarray(sig_pos, bool)
    carrier = sig_pos & ~(sym == BELOW).any(axis=0)   # no sample of the tile below its threshold
    L["carrier"] = carrier
    L["carrier_open"] = carrier & opened
    L["carried_open"] = ~carrier & opened & (open_edges == 0)
    # the carried state would open exactly on the run's first edge: the edge wins
    p_carried = run_from + np.maximum(0, n_T1 - np.asarray(n_samples, np.int64))
    L["carried_open_on_edge"] = sig_pos & (np.asarray(num_pulses) > NUM_PULSES_COMMAND) & (e_first >= 0) & \
        (e_first == p_carried) & (p_carried < nvalid)
    by_rise = opened & (open_edges > 0)
    L["short_open"] = by_rise & (n_T1 + 1 < 32)
    L["long_open"] = by_rise & (n_T1 + 1 >= 32)
    base = 32 * np.arange(edge_word.shape[0])[:, None]
    every_word_edged = ((base >= nvalid[None, :]) | edge_word).all(axis=0)
    L["long_open_no_free_word"] = L["long_open"] & every_word_edged
    L["word_skip"] = ~carrier & (n_T1 + 1 >= 64) & (nvalid - 1 - n_T1 > 0) & (e_first >= 0) & \
        ~L["carried_open"] & every_word_edged
    L["open_at_last"] = opened & (ret == nvalid - 1)
    L["carried_pulses_final"] = ~opened & ~invalid_seen & (np.asarray(num_pulses) > 0) & (valid_rises > 0)


# ------------------------------------------------------------------ parameters
def gate_pairs():
    """(n_T1, n_PW / 2, len_rn16, len_epc) of every defined configuration at decim 5 (the well-defined rates of
    tests/rate_rule.py, 0.4 and 0.6 MS/s), and the corners of the precondition half_pw <= 24"""
    from oracle.pyoracle import derive_cfg
    out = {}
    for r in list(GRID[well_defined(GRID)]) + [400000, 600000]:
        c = derive_cfg(adc_rate=int(r))
        if c.defined:
            out.setdefault((c.n_T1, c.n_PW // 2), (c.len_rn16, c.len_epc))
    for t1 in (30, 31, 32, 62, 63, 64):
        for hp in (0, 1, 23, 24):
            out.setdefault((t1, hp), (150, 822))
    return sorted(k + v for k, v in out.items())


def _choice(rng, options, n):
    options = np.asarray(options)
    return options[rng.integers(0, len(options), size=n)] if options.ndim == 1 else \
        options[np.arange(n), rng.integers(0, options.shape[1], size=n)]


def _symbols(level_low, starts, rng, p_equal):
    """levels -> symbols: an edge sample is decisive, the others are threshold-equal with probability p_equal"""
    decisive = np.where(level_low, BELOW, ABOVE).astype(np.int8)
    eq = (rng.random(level_low.shape, dtype=np.float32) < p_equal[:, None]) & ~starts
    return np.where(eq, NEITHER, decisive).astype(np.int8)


def _levels_from_durations(d, s0, P):
    """segments of durations d [N, K] (segment 0 low, then alternating) starting at s0 (may be negative) -> low
    level and segment-start flags over positions 0..P-1 (before s0 and after the last segment: high)"""
    N, K = d.shape
    b = s0[:, None] + np.concatenate([np.zeros((N, 1), np.int64), np.cumsum(d, axis=1)], axis=1)   # [N, K + 1]
    seg0 = (b <= 0).sum(axis=1) - 1          # the segment position 0 lies in (-1: before the train)
    tog = np.zeros((N, P + 1), np.int8)
    inside = (b > 0) & (b < P)
    r, c = np.nonzero(inside)
    tog[r, b[r, c]] = 1
    seg = seg0[:, None].astype(np.int32) + np.cumsum(tog[:, :P], axis=1, dtype=np.int32)
    low = (seg >= 0) & (seg < K) & (seg % 2 == 0)
    starts = tog[:, :P].astype(bool)
    starts[:, 0] |= (b == 0).any(axis=1)
    return low, starts, b


def make_cases(W, n, seed, pairs):
    """n single-tile cases: symbols [32 W, n] and the integer inputs of gate_closed_run"""
    rng = np.random.default_rng(seed)
    P = 32 * W
    pr = np.asarray(pairs, np.int64)[rng.integers(0, len(pairs), size=n)]
    n_T1, hp = pr[:, 0], pr[:, 1]
    # run start and end: word boundaries, the tile's last sample, a window closing anywhere
    run_from = _choice(rng, [0, 0, 1, 31, 32, 33, P - 1, -1], n)
    rnd = run_from < 0
    run_from[rnd] = rng.integers(0, P, size=rnd.sum())
    wb = 32 * rng.integers(1, W + 1, size=n)
    nv_opts = np.stack([np.full(n, P), np.full(n, P), run_from + 1, wb, wb - 1, wb + 1,
                        rng.integers(run_from + 1, P + 1), np.ones(n, np.int64)], axis=1)
    nvalid = _choice(rng, nv_opts, n)
    run_from[nvalid == 1] = 0
    nvalid = np.clip(nvalid, run_from + 1, P)
    # carried state
    sig_pos = rng.integers(0, 2, size=n)
    num_pulses = _choice(rng, [0, 5, 6, 7, 40], n)
    ns_opts = np.stack([np.zeros(n, np.int64), hp, hp + 1, n_T1 - 1, n_T1, n_T1 + 1, np.full(n, 1 << 20)], axis=1)
    n_samples = _choice(rng, ns_opts, n)
    kind = rng.integers(0, 8, size=n)     # 0-1 random level runs, 2-6 pulse trains, 7 carrier only
    p_equal = _choice(rng, [0.0, 0.0, 0.3, 0.9], n)
    # ---- random level runs at several densities
    sw = rng.random((n, P), dtype=np.float32) < _choice(rng, [0.01, 0.05, 0.2, 0.5], n)[:, None]
    low_r = ((rng.integers(0, 2, size=n)[:, None] + np.cumsum(sw, axis=1, dtype=np.int16)) & 1).astype(bool)
    starts_r = sw
    # ---- pulse trains: m pulses (low widths around half_pw, short highs), the quiet gap, more pulses.  The gap's rise
    # r is placed so that r + 1 + n_T1 (the opening) lands on a chosen position q.
    K = 64
    m = rng.integers(3, 10, size=n)
    lw = np.where(rng.random((n, K)) < 0.5, hp[:, None] + rng.integers(0, 2, size=(n, K)),
                  rng.integers(1, 2 * hp[:, None] + 4, size=(n, K)))
    hw = rng.integers(1, 3 * hp[:, None] + 9, size=(n, K))
    d = np.where(np.arange(K) % 2 == 0, lw, hw)
    d = np.maximum(d, 1)
    quiet = n_T1 + _choice(rng, [0, 1, 2, 2, 3], n) + np.where(rng.random(n) < 0.25, rng.integers(0, 40, size=n), 0)
    d[np.arange(n), 2 * m + 1] = quiet   # (2 m + 1: a high segment)
    q_opts = np.stack([nvalid - 1, nvalid - 1, nvalid, wb - 1, wb, wb + 1, np.full(n, P - 1), run_from + n_T1 + 1,
                       rng.integers(run_from, nvalid + 2)], axis=1)
    q = _choice(rng, q_opts, n)
    r = q - 1 - n_T1
    csum = np.concatenate([np.zeros((n, 1), np.int64), np.cumsum(d, axis=1)], axis=1)
    s0 = r - csum[np.arange(n), 2 * m + 1]
    low_t, starts_t, bnd = _levels_from_durations(d, s0, P)
    # a carried state that agrees with the train where the run starts, for half of the trains
    agree = (kind >= 2) & (kind <= 6) & (run_from > 0) & (rng.random(n) < 0.5)
    before = (bnd <= (run_from - 1)[:, None]).sum(axis=1) - 1
    last_b = np.where(before >= 0, bnd[np.arange(n), np.maximum(before, 0)], -(1 << 20))
    sig_pos = np.where(agree, (before < 0) | (before % 2 == 1) | (before > K - 1), sig_pos)
    n_samples = np.where(agree, np.minimum(run_from - 1 - last_b, 1 << 20), n_samples)
    # ---- carrier only: above bits or nothing at all (the packed kernel's one-vote path passes all-zero masks)
    low_c = np.zeros((n, P), bool)
    starts_c = rng.random((n, P), dtype=np.float32) < _choice(rng, [0.0, 0.0, 0.5, 1.0], n)[:, None]
    sel_r, sel_c = kind <= 1, kind == 7
    low = np.where(sel_r[:, None], low_r, np.where(sel_c[:, None], low_c, low_t))
    starts = np.where(sel_r[:, None], starts_r, np.where(sel_c[:, None], starts_c, starts_t))
    sym = _symbols(low, starts, rng, p_equal)
    sym[sel_c] = np.where(starts_c[sel_c], ABOVE, NEITHER)
    # glitches: a few single samples flipped to the other side of the threshold
    g = (rng.random((n, P), dtype=np.float32) < 0.004) & (kind[:, None] != 7)
    sym = np.where(g, np.where(sym == ABOVE, BELOW, ABOVE), sym).astype(np.int8)
    sym[np.arange(P)[None, :] >= nvalid[:, None]] = NEITHER        # masks are zero at and past nvalid
    return dict(sym=np.ascontiguousarray(sym.T), run_from=run_from, nvalid=nvalid, n_T1=n_T1, half_pw=hp,
                sig_pos=sig_pos.astype(np.int64), n_samples=n_samples, num_pulses=num_pulses)


def make_streams(W, n, T, seed, pairs):
    """n streams of T tiles: reader-like pulse trains with quiet gaps around n_T1, windows of the pair's lengths"""
    rng = np.random.default_rng(seed)
    P = 32 * W
    tot = P * T
    pr = np.asarray(pairs, np.int64)[rng.integers(0, len(pairs), size=n)]
    n_T1, hp, l0, l1 = pr.T
    K = tot // 3
    lw = np.where(rng.random((n, K)) < 0.5, hp[:, None] + rng.integers(0, 2, size=(n, K)),
                  rng.integers(1, 2 * hp[:, None] + 4, size=(n, K)))
    u = rng.random((n, K))
    hw = np.where(u < 0.12, n_T1[:, None] + rng.integers(-1, 4, size=(n, K)),
                  np.where(u < 0.15, rng.integers(1, l1[:, None] + 64), rng.integers(1, 3 * hp[:, None] + 9, size=(n, K))))
    d = np.maximum(np.where(np.arange(K) % 2 == 0, lw, hw), 1)
    low, starts, _ = _levels_from_durations(d, rng.integers(0, 64, size=n), tot)
    sym = _symbols(low, starts, rng, _choice(rng, [0.0, 0.3], n))
    nlast = np.where(rng.random(n) < 0.5, P, rng.integers(1, P + 1, size=n))
    n_total = (T - 1) * P + nlast
    sym[np.arange(tot)[None, :] >= n_total[:, None]] = NEITHER
    fresh = rng.random(n) < 0.5      # the reference's initial state, or a carried one
    sig_pos = np.where(fresh, 0, rng.integers(0, 2, size=n))
    num_pulses = np.where(fresh, 0, _choice(rng, [0, 5, 6, 7, 40], n))
    n_samples = np.where(fresh, 0, _choice(rng, [0, 1, 1 << 20], n))
    return dict(sym=np.ascontiguousarray(sym.T), n_total=n_total, nlast=nlast, n_T1=n_T1, half_pw=hp, l0=l0, l1=l1,
                sig_pos=sig_pos, n_samples=n_samples, num_pulses=num_pulses)


def pack_words(sym_t):
    """symbols [positions, n] -> (below, above) mask words [n, positions / 32] (bit p % 32 of word p / 32)"""
    n = sym_t.shape[1]
    out = []
    for v in (BELOW, ABOVE):
        bits = (sym_t.T == v).reshape(n, -1, 32)
        out.append(np.packbits(bits, axis=-1, bitorder="little").view("<u4")[..., 0].astype(np.uint32))
    return out


# ------------------------------------------------------------------ CPU: the replay against the restatement's gate
def _gate_inputs(o, y):
    """|y| (cabsf: the double-precision modulus rounded to float, gen2_oracle_cabsf) and the oracle's avg_ampl ->
    symbols"""
    g = o.gate(y, want_avg=True)
    yy = y.astype(np.complex64)
    a = np.sqrt(yy.real.astype(np.float64) ** 2 + yy.imag.astype(np.float64) ** 2).astype(np.float32)
    thr = (g["avg"] * THRESH_FRACTION).astype(np.float32)
    sym = np.where(a < thr, BELOW, np.where(a > thr, ABOVE, NEITHER)).astype(np.int8)
    return sym, g


def _replay_streams(items):
    """[(symbols, cfg)] -> replay of each as one stream from the reference's initial state"""
    n = len(items)
    P = max(s.size for s, _ in items)
    sym = np.zeros((P, n), np.int8)
    for i, (s, _) in enumerate(items):
        sym[:s.size, i] = s
    c = [cfg for _, cfg in items]
    z = np.zeros(n, np.int64)
    return replay(sym, z, np.array([s.size for s, _ in items]), np.array([x.n_T1 for x in c]),
                  np.array([x.n_PW // 2 for x in c]), z, z, z,
                  windows=(np.array([x.len_rn16 for x in c]), np.array([x.len_epc for x in c])), max_open=4096,
                  labels=False)


def test_replay_reproduces_the_restatements_gate(oracle, cfg1_iq):
    """the replay's openings = Oracle.gate's open_idx, window for window, on the recording, on every segment of the
    rate captures (all variants) and on the pulse-train captures"""
    from oracle.pyoracle import Oracle
    items, want = [], []
    sym, g = _gate_inputs(oracle, oracle.mf(cfg1_iq))
    items.append((sym, oracle.cfg))
    want.append(g)
    for adc, ntaps in RATES:
        o = Oracle(adc_rate=adc, ntaps=ntaps)
        for kw in RATE_VARIANTS.values():
            cap = rate_capture(adc, kw)
            iq = cap["iq"].numpy()
            for off, ln in zip(cap["segments"]["offset"], cap["segments"]["length"]):
                sym, g = _gate_inputs(o, o.mf(iq[int(off):int(off) + int(ln)]))
                items.append((sym, o.cfg))
                want.append(g)
    for adc, ntaps in PULSE_RATES:
        o = Oracle(adc_rate=adc, ntaps=ntaps)
        iq, segs = pulse_capture(adc, ntaps)
        for off, ln in zip(segs["offset"], segs["length"]):
            sym, g = _gate_inputs(o, o.mf(iq[int(off):int(off) + int(ln)]))
            items.append((sym, o.cfg))
            want.append(g)
    got = _replay_streams(items)
    total = 0
    for i, g in enumerate(want):
        k, n = int(got["n_open"][i]), g["n"]
        assert got["opens"][i, :n].tolist() == g["open_idx"].tolist(), i
        # Oracle.gate counts only the windows that closed; the replay also the last one when the segment ends inside it
        # (windows alternate RN16, EPC; a window holds its trigger and n_samples_to_ungate - 1 samples after it)
        assert k in (n, n + 1), (i, k, n)
        if k == n + 1:
            cfg, ny = items[i][1], items[i][0].size
            assert got["opens"][i, n] + (cfg.len_epc if n & 1 else cfg.len_rn16) > ny, (i, n)
        total += n
    assert total >= 3000 and want[0]["n"] >= 100, (total, want[0]["n"])


def pulse_widths(sym):
    """the reference's edges on one symbol sequence (signal_state follows the last sample below or above its threshold
    and starts NEG_EDGE) -> low-pulse widths (rise - fall: n_samples at the rise) and high gaps (fall - rise)"""
    p = np.arange(sym.size)
    last = np.maximum.accumulate(np.where(sym != NEITHER, p, -1))
    high = (last >= 0) & (sym[np.maximum(last, 0)] == ABOVE)
    e = np.nonzero(high[1:] != high[:-1])[0] + 1
    d = np.diff(e)
    is_rise = high[e[1:]]
    return d[is_rise], d[~is_rise]


def test_pack_words_layout():
    sym = np.zeros((64, 1), np.int8)
    sym[0, 0], sym[33, 0], sym[63, 0] = BELOW, ABOVE, BELOW
    lt, gt = pack_words(sym)
    assert lt.tolist() == [[1, 1 << 31]] and gt.tolist() == [[0, 2]]


def test_harness_build_helper(tmp_path):
    """the harness is built with the library's flags against the csrc it is given, and rebuilt when a header changes"""
    import ctypes
    import shutil
    from oracle import gate_harness as gh
    from gen2_uhf_rfid_reader_b200.build import NVCC_FLAGS
    csrc = tmp_path / "csrc"
    csrc.mkdir()
    shutil.copy(os.path.join(gh.CSRC, "rx_gate.cuh"), csrc)
    lib = str(tmp_path / "h.so")
    cmd = gh.command(lib, str(csrc))
    assert cmd[1:1 + len(NVCC_FLAGS)] == NVCC_FLAGS and "-fmad=false" in cmd and "arch=compute_90a,code=sm_90a" in cmd
    assert gh.stale(lib, str(csrc))
    if gh._nvcc() is None:
        pytest.skip("no nvcc on this machine")
    gh.build(lib=lib, csrc=str(csrc))
    assert not gh.stale(lib, str(csrc))
    t = os.path.getmtime(lib) + 10
    os.utime(csrc / "rx_gate.cuh", (t, t))
    assert gh.stale(lib, str(csrc))
    h = ctypes.CDLL(lib)
    assert h.gate_harness_masks and h.gate_harness_closed_run and h.gate_harness_stream


def test_generators_reach_every_rule():
    """the coverage the GPU tests assert, checked where it is cheap (smaller batch, same generators)"""
    pairs = [p[:2] for p in gate_pairs()]
    for W in (4, 8):
        c = make_cases(W, 40000, 7 + W, pairs)
        res = replay(c["sym"], c["run_from"], c["nvalid"], c["n_T1"], c["half_pw"], c["sig_pos"], c["n_samples"],
                     c["num_pulses"])
        counts = {k: int(v.sum()) for k, v in res["labels"].items() if k != "reopen_in_tile"}
        assert min(counts.values()) >= 20, (W, counts)


# ------------------------------------------------------------------ GPU: the harness
@pytest.fixture(scope="module")
def harness():
    from oracle import gate_harness
    return gate_harness.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(fn, *args):
    import torch
    torch.cuda.synchronize()
    err = fn(*[a.data_ptr() if hasattr(a, "data_ptr") else a for a in args])
    torch.cuda.synchronize()
    assert err == 0, "launch failed: cudaError %d" % err


def run_closed_run(h, W, c):
    import torch
    n = c["nvalid"].size
    lt, gt = pack_words(c["sym"])
    ins = np.stack([c["run_from"], c["nvalid"], c["n_T1"], c["half_pw"], c["sig_pos"], c["n_samples"],
                    c["num_pulses"]], axis=1).astype(np.int32)
    out = torch.zeros((n, 5), dtype=torch.int32, device="cuda")
    _run(h.gate_harness_closed_run, W, _dev(lt.view(np.int32)), _dev(gt.view(np.int32)), _dev(ins), out, n)
    return out.cpu().numpy()


def _first_mismatch(c, got, want, bad):
    i = int(np.nonzero(bad)[0][0])
    case = {k: (int(v[i]) if np.ndim(v) == 1 else None) for k, v in c.items()}
    s = c["sym"][:, i]
    case["sym"] = "".join(".-+"[v] for v in s[:case["nvalid"]])
    return "case %d of %d: %s\n  kernel %s, replay %s" % (i, int(bad.sum()), case, got[i].tolist(), want[:, i].tolist())


# minimum number of cases (per W, per million) that reach each rule
MIN_LABEL = {"carrier": 50000, "carrier_open": 5000, "carried_open": 20000, "carried_open_on_edge": 2000,
             "short_open": 2000, "long_open": 10000, "long_open_no_free_word": 300, "word_skip": 5000,
             "first_rise_invalid": 10000, "first_rise_at_half_pw": 2000, "pulse_half_pw": 20000,
             "pulse_half_pw_1": 20000, "fall_at_open": 5000, "open_at_last": 5000, "carried_pulses_open": 2000,
             "carried_pulses_final": 5000, "equal_high": 50000, "equal_low": 50000}


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_closed_run_matches_replay(harness, W):
    """524,288 single-tile cases per W: return value and all three state fields, exactly"""
    pairs = [p[:2] for p in gate_pairs()]
    counts = dict.fromkeys(MIN_LABEL, 0)
    n_all = 0
    for chunk in range(2):
        c = make_cases(W, 1 << 18, 1000 * W + chunk, pairs)
        got = run_closed_run(harness, W, c)
        res = replay(c["sym"], c["run_from"], c["nvalid"], c["n_T1"], c["half_pw"], c["sig_pos"], c["n_samples"],
                     c["num_pulses"])
        want = np.stack([res["ret"], res["sig_pos"], res["n_samples"], res["num_pulses"]])
        assert got[:, 4].all(), "lanes disagree"
        bad = (got[:, :4] != want.T).any(axis=1)
        assert not bad.any(), _first_mismatch(c, got, want, bad)
        for k in MIN_LABEL:
            counts[k] += int(res["labels"][k].sum())
        n_all += c["nvalid"].size
    short = {k: v for k, v in counts.items() if v * 1_000_000 < MIN_LABEL[k] * n_all}
    assert not short, "rules reached too rarely: %s" % short


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_closed_run_regression_cases(harness, W):
    """hand-made cases at the edges named in rx_gate.cuh, each with its expected result from the replay"""
    P = 32 * W
    cases = []

    def add(pattern, run_from=0, nvalid=P, n_T1=40, half_pw=2, sig_pos=1, n_samples=0, num_pulses=0):
        s = np.zeros(P, np.int8)
        for p, v in pattern:
            s[p] = v
        cases.append((s, run_from, nvalid, n_T1, half_pw, sig_pos, n_samples, num_pulses))

    def train(q, n_T1, half_pw, widths, gap_end=None):
        """low pulses of the given widths (fall-to-rise), highs of 3 samples, the last rise at q - 1 - n_T1"""
        r = q - 1 - n_T1
        pat = []
        for w in reversed(widths):
            pat += [(r, ABOVE), (r - w, BELOW)]
            r -= w + 3
        if gap_end is not None:
            pat.append((gap_end, BELOW))
        return [(p, v) for p, v in pat if 0 <= p < P]

    for t1 in (30, 31, 62, 63):
        for hpw in (0, 1, 3):
            ws = [hpw + 1] * 6
            add(train(P - 1, t1, hpw, ws), n_T1=t1, half_pw=hpw, sig_pos=1)          # opens at the last sample
            add(train(P, t1, hpw, ws), n_T1=t1, half_pw=hpw)                         # one sample short
            add(train(P - 5, t1, hpw, ws, gap_end=P - 5), n_T1=t1, half_pw=hpw)      # a fall at the opening
            add(train(P - 5, t1, hpw, [hpw] + ws[1:]), n_T1=t1, half_pw=hpw)         # one pulse exactly half_pw
            # five valid pulses: the carried count decides (opens at nvalid - 1 with one carried pulse, not without)
            add(train(P - 5, t1, hpw, ws[:5]), n_T1=t1, half_pw=hpw, num_pulses=1, nvalid=P - 4)
            add(train(P - 5, t1, hpw, ws[:5]), n_T1=t1, half_pw=hpw, num_pulses=0, nvalid=P - 4)
    add([(3, ABOVE)], sig_pos=0, n_samples=1, half_pw=2)                             # first rise, pulse began before
    add([(3, ABOVE)], sig_pos=0, n_samples=0, half_pw=3, run_from=1)
    add([(40, BELOW)], run_from=33, n_T1=20, n_samples=13, num_pulses=6)             # carried open on a fall
    sym = np.stack([c[0] for c in cases], axis=1)
    ints = [np.array([c[i] for c in cases], np.int64) for i in range(1, 8)]
    c = dict(sym=sym, run_from=ints[0], nvalid=ints[1], n_T1=ints[2], half_pw=ints[3], sig_pos=ints[4],
             n_samples=ints[5], num_pulses=ints[6])
    got = run_closed_run(harness, W, c)
    res = replay(sym, *ints)
    want = np.stack([res["ret"], res["sig_pos"], res["n_samples"], res["num_pulses"]])
    bad = (got[:, :4] != want.T).any(axis=1)
    assert not bad.any(), _first_mismatch(c, got, want, bad)
    # the trains that open at the last sample, and those whose carried pulse makes the sixth
    assert (res["ret"] >= 0).sum() == 24


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_streams_match_replay(harness, W):
    """64-tile streams through gate_closed_run the way the capture kernels call it, windows skipped by the ungate
    rule, second runs inside a tile: every opening and the final state"""
    import torch
    P, T, n, max_open = 32 * W, 64, 3000, 256
    s = make_streams(W, n, T, 77 + W, gate_pairs())
    lt, gt = pack_words(s["sym"])       # [stream][tile][word]
    nvalid = np.full((n, T), P, np.int32)
    nvalid[:, -1] = s["nlast"]
    ins = np.stack([s["n_T1"], s["half_pw"], s["l0"], s["l1"], s["sig_pos"], s["n_samples"], s["num_pulses"]],
                   axis=1).astype(np.int32)
    opens = torch.full((n, max_open), -1, dtype=torch.int32, device="cuda")
    meta = torch.zeros((n, 7), dtype=torch.int32, device="cuda")
    _run(harness.gate_harness_stream, W, _dev(lt.view(np.int32)), _dev(gt.view(np.int32)), _dev(nvalid), _dev(ins),
         T, opens, max_open, meta, n)
    opens, meta = opens.cpu().numpy(), meta.cpu().numpy()
    z = np.zeros(n, np.int64)
    res = replay(s["sym"], z, s["n_total"], s["n_T1"], s["half_pw"], s["sig_pos"], s["n_samples"], s["num_pulses"],
                 windows=(s["l0"], s["l1"]), max_open=max_open, tile=P)
    assert meta[:, 5].all() and meta[:, 6].all(), "lanes disagree or a tile did not terminate"
    assert (res["n_open"] <= max_open).all()
    for i in range(n):
        k = int(res["n_open"][i])
        want = [int(res["n_open"][i]), int(res["sig_pos"][i]), int(res["n_samples"][i]), int(res["num_pulses"][i]),
                int(res["gate_open"][i])]
        assert meta[i, :5].tolist() == want and opens[i, :k].tolist() == res["opens"][i, :k].tolist(), \
            "stream %d (n_T1 %d, half_pw %d): kernel %s %s, replay %s %s" % (
                i, s["n_T1"][i], s["half_pw"][i], meta[i, :5].tolist(), opens[i, :k].tolist(), want,
                res["opens"][i, :k].tolist())
    assert res["n_open"].sum() >= n
    assert res["labels"]["reopen_in_tile"].sum() >= n // 40


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_masks_match_float32_comparison(harness, W):
    """gate_masks: bit p of the below / above word is a < 0.75 avg / a > 0.75 avg in float32, nothing at or past nvalid;
    samples exactly at the threshold are neither"""
    import torch
    rng = np.random.default_rng(5 + W)
    P, n = 32 * W, 1 << 16
    avg = (10.0 ** rng.uniform(-4, 1, size=(n, P))).astype(np.float32)
    thr = (avg * THRESH_FRACTION).astype(np.float32)
    k = rng.integers(0, 5, size=(n, P))
    a = np.select([k == 0, k == 1, k == 2],
                  [thr, np.nextafter(thr, np.float32(np.inf)), np.nextafter(thr, np.float32(0))],
                  (thr * rng.uniform(0.5, 1.5, size=(n, P))).astype(np.float32)).astype(np.float32)
    nvalid = np.where(rng.random(n) < 0.5, P, rng.integers(1, P + 1, size=n)).astype(np.int32)
    lt = torch.zeros((n, 32), dtype=torch.int32, device="cuda")
    gt = torch.zeros((n, 32), dtype=torch.int32, device="cuda")
    _run(harness.gate_harness_masks, W, _dev(avg), _dev(a), _dev(nvalid), lt, gt, n)
    inside = np.arange(P)[None, :] < nvalid[:, None]
    sym = np.where(inside & (a < avg * THRESH_FRACTION), BELOW,
                   np.where(inside & (a > avg * THRESH_FRACTION), ABOVE, NEITHER)).astype(np.int8)
    wl, wg = pack_words(np.ascontiguousarray(sym.T))
    lane = np.arange(32) % W
    assert (lt.cpu().numpy().view(np.uint32) == wl[:, lane]).all()
    assert (gt.cpu().numpy().view(np.uint32) == wg[:, lane]).all()
    assert (inside & (a == thr)).sum() >= n * P // 10


# ------------------------------------------------------------------ pulse-train captures through every capture kernel
# The call sites hold gate logic of their own that the harness does not run: the packed kernel's one-vote quiet test
# and its second closed run in a tile (with the DC recompute after a window), the split kernel's skip of tiles inside a
# window.  These captures (make_golden.pulse_capture) put pulse widths and quiet gaps at the gate's bounds.
def test_pulse_captures_straddle_the_gate_bounds():
    """after the boxcar, the reference's edges (from the restatement's avg_ampl and |y|) include low pulses exactly
    n_PW / 2 and n_PW / 2 + 1 wide and quiet gaps exactly n_T1 and n_T1 + 1 long, at every rate; and the restatement
    decodes the captures as the reference's blocks did"""
    from oracle.pyoracle import Oracle
    from conftest import records_equal
    with np.load(os.path.join(GOLDEN, "reference_pulses.npz")) as z:
        ref = {k: z[k] for k in z.files}
    for adc, ntaps in PULSE_RATES:
        o = Oracle(adc_rate=adc, ntaps=ntaps)
        iq, segs = pulse_capture(adc, ntaps)
        widths, gaps = [], []
        for off, ln in zip(segs["offset"], segs["length"]):
            w, g = pulse_widths(_gate_inputs(o, o.mf(iq[int(off):int(off) + int(ln)]))[0])
            widths.append(w)
            gaps.append(g)
        widths, gaps = np.concatenate(widths), np.concatenate(gaps)
        hp, t1 = o.cfg.n_PW // 2, o.cfg.n_T1
        # (a pulse is at least one sample wide: at half_pw = 0 only half_pw + 1 can occur)
        for v in ([hp, hp + 1] if hp > 0 else [1]):
            assert (widths == v).sum() >= 3, (adc, v)
        for v in (t1, t1 + 1):
            assert (gaps == v).sum() >= 3, (adc, v)
        key = "p%d_t%d" % (adc, ntaps)
        orecs, ocounts, _ = o.decode_segments(iq, segs, max_per_seg=PULSE_MAX_WINDOWS)
        assert ocounts.tolist() == ref[key + "_counts"].tolist() and ocounts.sum() >= 3 * segs.size, adc
        assert not records_equal(orecs, ref[key + "_records"]), adc


# (id, adc rate, taps, environment, the capture kernel that must decode it)
PULSE_KERNELS = [
    ("pack_2000_g1", 2000000, 25, {"RFID_B200_PACK_G": "1"}, "rx_pack_kernel"),
    ("pack_2000_g8", 2000000, 25, {"RFID_B200_PACK_G": "8"}, "rx_pack_kernel"),
    ("pack_1200_g1", 1200000, 25, {"RFID_B200_PACK_G": "1"}, "rx_pack_kernel"),
    ("pack_1200_g8", 1200000, 25, {"RFID_B200_PACK_G": "8"}, "rx_pack_kernel"),
    ("split_2000", 2000000, 25, {"RFID_B200_KERNEL": "split"}, "rx_fused_split_kernel"),
    ("split_400", 400000, 25, {}, "rx_fused_split_kernel"),
    ("split_1000", 1000000, 25, {}, "rx_fused_split_kernel"),
    ("split_2400", 2400000, 25, {}, "rx_fused_split_kernel"),
    ("fused_2600", 2600000, 25, {}, "rx_fused_kernel"),
    ("fused_4000", 4000000, 50, {}, "rx_fused_kernel"),
    ("fused_8000", 8000000, 100, {}, "rx_fused_kernel"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PULSE_KERNELS, ids=[c[0] for c in PULSE_KERNELS])
def test_pulse_captures_through_every_capture_kernel(case, monkeypatch):
    """window counts and records, bit for bit, against the reference's blocks (reference_pulses.npz) and the
    restatement"""
    from conftest import records_equal
    from gen2_uhf_rfid_reader_b200 import capi
    from oracle.pyoracle import Oracle
    from test_rate_parity import _kernel_names
    _, adc, ntaps, env, kernel = case
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rx = capi.Gen2Rx(adc_rate=adc, ntaps=ntaps)
    iq, segs = pulse_capture(adc, ntaps)
    assert _kernel_names(lambda: rx.decode_capture_host(iq, segs, max_windows=PULSE_MAX_WINDOWS)) == {kernel}
    recs, counts = rx.decode_capture_host(iq, segs, max_windows=PULSE_MAX_WINDOWS)
    key = "p%d_t%d" % (adc, ntaps)
    with np.load(os.path.join(GOLDEN, "reference_pulses.npz")) as z:
        assert counts.tolist() == z[key + "_counts"].tolist()
        bad = records_equal(recs, z[key + "_records"])
        assert not bad, "fields differ from the reference: %s" % bad
    orecs, ocounts, _ = Oracle(adc_rate=adc, ntaps=ntaps).decode_segments(iq, segs, max_per_seg=PULSE_MAX_WINDOWS)
    assert counts.tolist() == ocounts.tolist()
    bad = records_equal(recs, orecs)
    assert not bad, "fields differ from the restatement: %s" % bad
