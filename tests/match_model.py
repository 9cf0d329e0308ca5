"""numpy restatement of the EPC match rule (include/rfid_b200.h, csrc/rx_match.cuh) -- test infrastructure.

Per stored window: an RN16 window is NOT_EPC; an EPC window whose CRC passes, or whose fix is RECOVERED, ALREADY_READ;
otherwise it is attempted.  It is SKIPPED when crc_ok != 0 or S1 = sum |r_j| (the quality rule's projections and lane
order) is 0 or not finite.  Else q_j = min(127, rint(|r_j| * 16 / (S1 / 128))), s_j = r_j > 0, and entry k costs
D_k = sum q_j [s_j != c_kj] with c_k the signs of frame k (c_kj = c_k,j-1 xor bit_kj, c_k,-1 = 1).  k* = argmin (lowest
index on ties), D1, D2 the two smallest of the multiset; MATCHED iff D1 <= 16 max_cost and D2 - D1 >= 16 min_margin,
AMBIGUOUS iff only the first, else NO_MATCH.
"""
import numpy as np

import quality_model as qm
import recover_model as rm

f32, f64 = np.float32, np.float64

ALREADY_READ, MATCHED, AMBIGUOUS, NO_MATCH, SKIPPED, NOT_EPC = range(6)
EPC_MATCH_DTYPE = np.dtype([("status", "<i4"), ("entry", "<i4"), ("cost", "<i4"), ("runner_up", "<i4"),
                            ("n_diff", "<i4"), ("reserved", "<i4", (3,))])
MATCH_COUNT_DTYPE = np.dtype([("matched", "<i4"), ("first_slot", "<i4"), ("last_slot", "<i4"), ("reserved", "<i4")])
DEFAULT_MAX_COST, DEFAULT_MIN_MARGIN = 12.0, 4.0
INT32_MAX = 2 ** 31 - 1
FIX_RECOVERED = 1


def thresholds(max_cost=DEFAULT_MAX_COST, min_margin=DEFAULT_MIN_MARGIN):
    """the host's thresholds in reliability steps: 16 * (double) of the float settings"""
    return float(f32(max_cost)) * 16.0, float(f32(min_margin)) * 16.0


def codeword_signs(frames):
    """frames uint8 [K, 16] -> codeword signs uint8 [K, 128] in {0, 1} (the decoder's differential FM0 rule)"""
    b = np.unpackbits(np.asarray(frames, dtype=np.uint8).reshape(-1, 16), axis=1).astype(bool)
    ones = np.ones((b.shape[0], 1), dtype=bool)
    return np.logical_xor.accumulate(np.concatenate([ones, b], axis=1), axis=1)[:, 1:].astype(np.uint8)


def reliabilities(r):
    """projections float32 [..., 128] -> (q int64 [..., 128], s bool [..., 128], ok bool [...]): ok is False where S1
    is 0 or not finite (SKIPPED)"""
    r = np.asarray(r, dtype=f32)
    a = np.abs(r.astype(f64))
    lead = r.shape[:-1]
    s1 = np.array([qm.lane_sum(x) for x in a.reshape(-1, 128)]).reshape(lead)
    ok = np.isfinite(s1) & (s1 > 0)
    m = np.where(ok, s1 / 128.0, 1.0)
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.minimum(127.0, np.rint((a * 16.0) / m[..., None]))
    q = np.where(ok[..., None], q, 0).astype(np.int64)
    return q, r > 0, ok


def costs(q, s, codewords):
    """D [N, K] = sum_j q_j [s_j != c_kj], directly"""
    q = np.asarray(q, dtype=np.int64)
    return (q[:, None, :] * (np.asarray(s, dtype=bool)[:, None, :] != np.asarray(codewords, dtype=bool)[None])).sum(-1)


def costs_gemm(q, s, codewords):
    """D [N, K] = A + u . c^T with u_j = q_j (1 - 2 s_j), A = sum q_j s_j: the kernel's int8 product"""
    q = np.asarray(q, dtype=np.int64)
    s = np.asarray(s, dtype=np.int64)
    u = (q * (1 - 2 * s)).astype(f64)   # float64 products and sums of integers below 2^53 are exact
    return (q * s).sum(-1)[:, None] + np.rint(u @ np.asarray(codewords, dtype=f64).T).astype(np.int64)


def top2(D):
    """D [N, K] -> (k* [N], D1 [N], D2 [N]): lowest index on ties, D2 the multiset's second smallest (INT32_MAX, K = 1)"""
    N, K = D.shape
    if K == 0:
        return np.full(N, -1), np.full(N, INT32_MAX), np.full(N, INT32_MAX)
    k1 = np.argmin(D, axis=1)            # the first minimum
    d1 = D[np.arange(N), k1]
    if K == 1:
        return k1, d1, np.full(N, INT32_MAX)
    d2 = np.partition(D, 1, axis=1)[:, 1]
    return k1, d1, d2


def decide(D, n_diff, max_cost=DEFAULT_MAX_COST, min_margin=DEFAULT_MIN_MARGIN):
    """attempted windows: D [N, K] and their n_diff function -> EPC_MATCH_DTYPE [N]"""
    N, K = D.shape
    out = np.zeros(N, dtype=EPC_MATCH_DTYPE)
    k1, d1, d2 = top2(D)
    out["entry"], out["cost"], out["runner_up"] = k1, d1, d2
    if K == 0:
        out["status"], out["n_diff"] = NO_MATCH, -1
        return out
    c16, m16 = thresholds(max_cost, min_margin)
    first = d1.astype(f64) <= c16
    second = (d2.astype(np.int64) - d1).astype(f64) >= m16
    out["status"] = np.where(first, np.where(second, MATCHED, AMBIGUOUS), NO_MATCH)
    out["n_diff"] = n_diff(k1)
    return out


def _not_attempted(status):
    out = np.zeros((), dtype=EPC_MATCH_DTYPE)
    out["status"] = status
    out["entry"] = out["cost"] = out["runner_up"] = out["n_diff"] = -1
    return out


def live_count(max_dict, n_dict=None):
    return max_dict if n_dict is None else min(max(int(n_dict), 0), max_dict)


def match_projections(r, dictionary, max_cost=DEFAULT_MAX_COST, min_margin=DEFAULT_MIN_MARGIN):
    """attempted windows given by their projections r float32 [N, 128] against frames [K, 16] -> EPC_MATCH_DTYPE [N]
    (SKIPPED where S1 is 0 or not finite)"""
    r = np.asarray(r, dtype=f32).reshape(-1, 128)
    q, s, ok = reliabilities(r)
    cw = codeword_signs(dictionary)
    out = np.zeros(r.shape[0], dtype=EPC_MATCH_DTYPE)
    if (~ok).any():
        out[~ok] = _not_attempted(SKIPPED)
    if ok.any():
        D = costs_gemm(q[ok], s[ok], cw)
        sk = s[ok]
        out[ok] = decide(D, lambda k: (sk != cw[k].astype(bool)).sum(-1) if cw.shape[0] else -1, max_cost, min_margin)
    return out


def match(windows, recs, counts, dictionary, fixes=None, n_dict=None, adc_rate=2_000_000,
          max_cost=DEFAULT_MAX_COST, min_margin=DEFAULT_MIN_MARGIN, decim=5):
    """the device call's layout: windows [nseg, max_windows, len_epc] complex64, recs RESULT_DTYPE [nseg, max_windows],
    fixes EPC_FIX_DTYPE or None, dictionary uint8 [max_dict, 16] -> (EPC_MATCH_DTYPE [nseg, max_windows] zero beyond
    the stored records, MATCH_COUNT_DTYPE [max_dict])"""
    _, n_f, _, len_epc = qm.derived(adc_rate, decim)
    dictionary = np.asarray(dictionary, dtype=np.uint8).reshape(-1, 16)
    K = live_count(dictionary.shape[0], n_dict)
    nseg, mw = recs.shape
    out = np.zeros((nseg, mw), dtype=EPC_MATCH_DTYPE)
    slots, rows = [], []
    for s in range(nseg):
        for k in range(min(max(int(counts[s]), 0), mw)):
            rec = recs[s, k]
            if int(rec["kind"]) != 1:
                out[s, k] = _not_attempted(NOT_EPC)
            elif int(rec["crc_ok"]) == 1 or (fixes is not None and int(fixes[s, k]["status"]) == FIX_RECOVERED):
                out[s, k] = _not_attempted(ALREADY_READ)
            elif int(rec["crc_ok"]) != 0:
                out[s, k] = _not_attempted(SKIPPED)
            else:
                slots.append((s, k))
                rows.append(rm.epc_projections(windows[s, k], rec, n_f, len_epc))
    if rows:
        res = match_projections(np.stack(rows), dictionary[:K], max_cost, min_margin)
        for (s, k), v in zip(slots, res):
            out[s, k] = v
    return out, match_counts(out, dictionary.shape[0])


def decoys(truth, n, rng, weights=range(4, 17)):
    """(frames uint8 [n, 16], sign distances [n]): CRC-valid frames at sign distance w from truth, w cycling through
    `weights`, PC length field intact -- truth with a sign set flipped whose syndrome columns (recover_model.SIGN_COL:
    CRC-16 and length field) XOR to zero.  A table of sign pairs completes random (w - 2)-sets."""
    col = rm.SIGN_COL
    pairs = {}
    for a in range(128):
        for b in range(a + 1, 128):
            pairs.setdefault(int(col[a] ^ col[b]), []).append((a, b))
    truth_s = codeword_signs(truth)[0].astype(bool)
    out, dist = [], []
    weights = list(weights)
    while len(out) < n:
        w = weights[len(out) % len(weights)]
        base = rng.choice(128, size=w - 2, replace=False)
        x = int(np.bitwise_xor.reduce(col[base]))
        cands = [p for p in pairs.get(x, []) if p[0] not in base and p[1] not in base]
        if not cands:
            continue
        s = truth_s.copy()
        s[np.concatenate([base, cands[rng.integers(len(cands))]])] ^= True
        f = np.packbits((s ^ np.concatenate([[True], s[:-1]])).astype(np.uint8))
        assert rm.syndrome(f) == 0 and (f[0] >> 3) == (np.asarray(truth)[0] >> 3)
        out.append(f)
        dist.append(w)
    return np.array(out), np.array(dist)


def match_counts(out, max_dict):
    """per-entry counts of the MATCHED windows of EPC_MATCH_DTYPE [nseg, max_windows] (slot = s * max_windows + k)"""
    cnt = np.zeros(max_dict, dtype=MATCH_COUNT_DTYPE)
    cnt["first_slot"] = cnt["last_slot"] = -1
    flat = out.reshape(-1)
    for i in np.nonzero(flat["status"] == MATCHED)[0]:
        e = int(flat[i]["entry"])
        c = cnt[e]
        c["matched"] += 1
        c["first_slot"] = i if c["first_slot"] < 0 else min(int(c["first_slot"]), i)
        c["last_slot"] = max(int(c["last_slot"]), i)
        cnt[e] = c
    return cnt
