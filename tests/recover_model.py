"""numpy restatement of the EPC recovery rule (include/rfid_b200.h, csrc/rx_recover.cuh) -- test infrastructure.

Per stored window: an RN16 window is NOT_EPC, an EPC window whose CRC passes CRC_OK, a failing one SKIPPED unless its
quality record has 128 decisions and snr >= min_snr_ratio.  Otherwise the projections r_j (quality_model's positions
and projections), reliabilities |r_j|, and the P least reliable sign positions by (|r_j|, j); every flip set F of 1..W of
them is a candidate (flipping sign j flips bits j and j + 1), and a candidate passes iff its CRC-16 and its PC length
field (00110) check.  Exactly one passer: RECOVERED, with the corrected bits, |F| and cost = sum |r_j| over F (ascending
j) / (S1 / 128); two or more AMBIGUOUS, none FAILED.  Candidates are tested through the syndrome, which is affine in
the bits (the tests check it against the bit rule).
"""
import functools
import itertools
from math import comb

import numpy as np

import quality_model as qm

f32, f64 = np.float32, np.float64

CRC_OK, RECOVERED, AMBIGUOUS, FAILED, SKIPPED, NOT_EPC = range(6)
EPC_FIX_DTYPE = np.dtype([("status", "<i4"), ("n_flips", "<i4"), ("n_pass", "<i4"), ("cost", "<f4"),
                          ("bits", "u1", (16,))])
DEFAULT_P, DEFAULT_W, DEFAULT_MIN_SNR_DB = 12, 4, 7.0
PC_LENGTH = 0b00110   # 6 words: the 96-bit EPC a 128-bit window holds


def snr_ratio(min_snr_db=DEFAULT_MIN_SNR_DB):
    """the host's linear threshold: 10^(dB/10) in double of the float setting"""
    return 10.0 ** (float(f32(min_snr_db)) / 10.0)


def n_candidates(P=DEFAULT_P, W=DEFAULT_W):
    return sum(comb(P, k) for k in range(1, W + 1))


def false_accept_bound(P=DEFAULT_P, W=DEFAULT_W):
    """C * 2^-21: each candidate passes a window whose true error set is not a candidate with probability about 2^-21"""
    return n_candidates(P, W) * 2.0 ** -21


# ------------------------------------------------------------------ the syndrome
def _crc_bits(crc, one_at):
    for m in range(112):
        fb = ((crc >> 15) & 1) ^ (1 if m == one_at else 0)
        crc = (crc << 1) & 0xFFFF
        if fb:
            crc ^= 0x1021
    return crc


def _columns():
    col = np.zeros(128, dtype=np.uint32)
    for j in range(128):
        s = _crc_bits(0, j) if j < 112 else 1 << (127 - j)
        if j < 5:
            s |= 1 << (20 - j)
        col[j] = s
    zero = ((~_crc_bits(0xFFFF, -1)) & 0xFFFF) | (PC_LENGTH << 16)
    return col, np.uint32(zero)


#: syndrome column of message bit j, and the syndrome of the all-zero window
BIT_COL, ZERO = _columns()
#: syndrome column of sign j: flipping it flips bits j and j + 1 (j = 127: bit 127 only)
SIGN_COL = BIT_COL ^ np.concatenate([BIT_COL[1:], np.zeros(1, dtype=np.uint32)])


def syndrome(bits):
    """linear form: bits uint8 [..., 16] (MSB first) -> uint32 [...]"""
    b = np.unpackbits(np.asarray(bits, dtype=np.uint8), axis=-1).astype(bool)
    return np.bitwise_xor.reduce(np.where(b, BIT_COL, np.uint32(0)), axis=-1) ^ ZERO


def syndrome_direct(frame):
    """the bit rule: CRC-16 of bytes 0..13 (synth.crc16_gen2) xor bytes 14..15, PC bits 0..4 xor 00110 at bits 16..20"""
    from gen2_uhf_rfid_reader_b200 import synth
    b = bytes(bytearray(np.asarray(frame, dtype=np.uint8)))
    return (synth.crc16_gen2(b[:14]) ^ int.from_bytes(b[14:16], "big")) | (((b[0] >> 3) ^ PC_LENGTH) << 16)


@functools.lru_cache(maxsize=None)
def combos(P, W):
    """every flip set of 1..W of the P ranks, padded with P (a zero column): int [C, W]"""
    rows = [list(c) + [P] * (W - k) for k in range(1, W + 1) for c in itertools.combinations(range(P), k)]
    return np.array(rows, dtype=np.int64).reshape(-1, W)


def candidate_syndromes(rho, syn, P, W):
    """rho float32 [N, 128], syn uint32 [N] -> (order int [N, P]: the P least reliable sign positions by (rho, j),
    syndromes uint32 [N, C] of the candidates combos(P, W))"""
    order = np.argsort(rho, axis=1, kind="stable")[:, :P]
    cols = np.concatenate([SIGN_COL[order], np.zeros((rho.shape[0], 1), dtype=np.uint32)], axis=1)
    cb = combos(P, W)
    s = np.repeat(np.asarray(syn, dtype=np.uint32)[:, None], cb.shape[0], axis=1)
    for t in range(W):
        s ^= cols[:, cb[:, t]]
    return order, s


def n_pass_batch(rho, bits, P=DEFAULT_P, W=DEFAULT_W, chunk=8192):
    """passing candidates of many attempted windows: rho float32 [N, 128], bits uint8 [N, 16] -> int [N]"""
    out = np.zeros(rho.shape[0], dtype=np.int64)
    for i in range(0, rho.shape[0], chunk):
        _, s = candidate_syndromes(rho[i:i + chunk], syndrome(bits[i:i + chunk]), P, W)
        out[i:i + chunk] = (s == 0).sum(axis=1)
    return out


# ------------------------------------------------------------------ the rule
def decide(r, bits, P=DEFAULT_P, W=DEFAULT_W):
    """an attempted window: projections r float32 [128], the record's bits uint8 [16] -> EPC_FIX_DTYPE scalar"""
    out = np.zeros((), dtype=EPC_FIX_DTYPE)
    out["bits"] = bits
    out["cost"] = np.nan
    r = np.asarray(r, dtype=f32)
    rho = np.abs(r)
    order, s = candidate_syndromes(rho[None, :], syndrome(bits)[None], P, W)
    passing = np.nonzero(s[0] == 0)[0]
    out["n_pass"] = passing.size
    if passing.size != 1:
        out["status"] = FAILED if passing.size == 0 else AMBIGUOUS
        return out
    ranks = combos(P, W)[passing[0]]
    F = np.sort(order[0][ranks[ranks < P]])
    flipped = 0.0
    for j in F:
        flipped += float(rho[j])
    mean = qm.lane_sum(np.abs(r.astype(f64))) / 128.0
    with np.errstate(divide="ignore", invalid="ignore"):
        out["cost"] = qm.canonical(f64(flipped) / f64(mean))
    b = np.unpackbits(np.asarray(bits, dtype=np.uint8))
    for j in F:
        b[j] ^= 1
        if j < 127:
            b[j + 1] ^= 1
    out["bits"] = np.packbits(b)
    out["status"], out["n_flips"] = RECOVERED, F.size
    return out


def epc_projections(w, rec, n_f, len_epc):
    """r_j of an EPC window as the quality rule computes them (samples outside [0, n) are 0)"""
    n = max(0, min(int(rec["length"]), len_epc))
    w = np.concatenate([np.ascontiguousarray(w[:n], dtype=np.complex64), np.zeros(1, dtype=np.complex64)])
    h = np.complex64(complex(f32(rec["h_re"]), f32(rec["h_im"])))
    a, b, _, _ = qm.positions(1, int(rec["sync_index"]), rec["T"], f32(n_f), 0)
    return qm.projections(w, n, a, b, h)


def recover_window(w, rec, q, n_f, len_epc, P=DEFAULT_P, W=DEFAULT_W, min_ratio=None):
    """one EPC_FIX_DTYPE record of window samples w (complex64), its RESULT_DTYPE record and its QUALITY_DTYPE record"""
    min_ratio = snr_ratio() if min_ratio is None else min_ratio
    out = np.zeros((), dtype=EPC_FIX_DTYPE)
    out["bits"] = rec["bits"]
    out["cost"] = np.nan
    if int(rec["kind"]) != 1:
        out["status"] = NOT_EPC
    elif int(rec["crc_ok"]) == 1:
        out["status"] = CRC_OK
    elif not (int(q["n_decisions"]) == 128 and float(q["snr"]) >= min_ratio):
        out["status"] = SKIPPED
    else:
        out = decide(epc_projections(w, rec, n_f, len_epc), rec["bits"], P, W)
    return out


def recover(windows, recs, counts, quality, adc_rate=2_000_000, P=DEFAULT_P, W=DEFAULT_W,
            min_snr_db=DEFAULT_MIN_SNR_DB, decim=5):
    """the device call's layout: windows [nseg, max_windows, len_epc] complex64, recs RESULT_DTYPE and quality
    QUALITY_DTYPE [nseg, max_windows] -> EPC_FIX_DTYPE [nseg, max_windows], zero beyond the stored records"""
    _, n_f, _, len_epc = qm.derived(adc_rate, decim)
    mr = snr_ratio(min_snr_db)
    nseg, mw = recs.shape
    out = np.zeros((nseg, mw), dtype=EPC_FIX_DTYPE)
    for s in range(nseg):
        for k in range(min(max(int(counts[s]), 0), mw)):
            out[s, k] = recover_window(windows[s, k], recs[s, k], quality[s, k], n_f, len_epc, P, W, mr)
    return out


def sign_errors(r, frame):
    """the sign positions whose decision differs from the true frame's (uint8 [16]): signs s_j = s_(j-1) xor bit_j,
    s_(-1) = 1"""
    b = np.unpackbits(np.asarray(frame, dtype=np.uint8)).astype(bool)
    true_sign = np.logical_xor.accumulate(np.concatenate([[True], b]))[1:]
    return np.nonzero((np.asarray(r) > 0) != true_sign)[0]
