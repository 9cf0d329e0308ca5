"""Which sample rates the reference decoder handles without reading past its window, evaluated in plain numpy float32.

The reference's tag decoder (tag_decoder_impl.cc) derives every read index from the float n_samples_TAG_BIT, while the
gate sizes the windows from its integer truncation (gate_impl.cc:115,121).  Where the two differ the EPC symbol-period
search and bit decisions read past the end of the EPC window, and an RN16 window can end before its 32 half-bits.  A
configuration is *well defined* when, for every sync index the preamble search can return, none of that happens.

This is a second, independent statement of the rule in csrc/rfid_b200.cu (derive_config) and oracle/gen2_oracle.c
(gen2_oracle_make_cfg).  It evaluates every rate of a grid at once and, where a read index grows with a loop counter
(float rounding is monotone), only the loop's last iteration.
"""
import numpy as np

f32 = np.float32


def derived(adc_rate, decim=5):
    """gate_impl.cc:48-53,115,121 and tag_decoder_impl.cc:60 with the reference's types, for an array of rates"""
    sr = np.asarray(adc_rate, dtype=np.int64) // decim
    n_i = (25.0 * (sr / 1e6)).astype(np.int64)                      # int * (int / double), truncated
    n_f = ((f32(25.0) * sr.astype(f32)).astype(np.float64) / 1e6).astype(f32)  # float * int / double -> float
    return n_i, n_f, 25 * n_i, 137 * n_i


def well_defined(adc_rate, decim=5):
    """bool array: the reference decoder stays inside its windows at these rates"""
    n_i, n_f, len_rn16, len_epc = derived(adc_rate, decim)
    ok = n_i >= 1
    sync_range = np.ceil(1.5 * n_f.astype(np.float64)).astype(np.int64)   # i < 1.5 * n  (:85)
    half = (n_f / f32(2)).astype(f32)
    # tag_sync: in[(int)(i + j*n/2)] for i < sync_range, j < 12; h_est's taps (:103) are among them
    last_sync = ((sync_range - 1).astype(f32) + (f32(11) * n_f).astype(f32) / f32(2)).astype(f32).astype(np.int64)
    ok &= last_sync < len_rn16
    # tag_detection_EPC (:151-152,161,166,173): the 20 candidate half-periods
    n64 = n_f.astype(np.float64)
    lo = (n64 / 2.0 - n64 / 2.0 / 100).astype(f32)
    hi = (n64 / 2.0 + n64 / 2.0 / 100).astype(f32)
    t = np.arange(20, dtype=f32)[:, None]
    steps = (lo + ((t * (hi - lo)).astype(f32) / f32(19)).astype(f32)).astype(f32)       # [20, rates]
    for s in range(int(sync_range.max())):
        live = s < sync_range
        index = ((f32(s) + (f32(6) * n_f).astype(f32)).astype(f32) + half).astype(f32).astype(np.int64)  # :107
        # RN16 half-bits (:237-253): float j from index in steps of n/2 while j < ninput; the 32nd must be taken
        j = index.astype(f32)
        got = np.zeros(n_f.shape, dtype=bool)
        reads_ok = np.ones(n_f.shape, dtype=bool)
        for _ in range(32):
            inside = j < len_rn16.astype(f32)
            k = np.floor(j.astype(np.float64) + 0.5).astype(np.int64)      # round(): halves away from zero
            reads_ok &= ~inside | (k < len_rn16)
            got = inside
            j = (j + half).astype(f32)
            if not inside.any():
                break
        # energy search: magn_squared_samples[(int)(i * step + index)] for i < 256
        e_last = ((f32(255) * steps).astype(f32) + index.astype(f32)).astype(f32).astype(np.int64).max(axis=0)
        # bit decisions at T = step: in[(int)(j*(2T) + index)], in[(int)(j*2*T + T + index)] for j < 128
        b_last = ((((f32(254) * steps).astype(f32) + steps).astype(f32)) + index.astype(f32)).astype(f32)
        b_last = b_last.astype(np.int64).max(axis=0)
        a_last = ((f32(127) * (f32(2) * steps).astype(f32)).astype(f32) + index.astype(f32)).astype(f32)
        a_last = a_last.astype(np.int64).max(axis=0)
        ok &= ~live | (got & reads_ok & (e_last < len_epc) & (a_last < len_epc) & (b_last < len_epc))
    return ok


GRID = np.arange(1_000_000, 8_000_001, 1000, dtype=np.int64)
