"""numpy restatement of the tag inventory report (include/rfid_b200.h, csrc/rx_report.cuh) -- test infrastructure.

Stored slot i = s * max_windows + k, k < min(max(count[s], 0), max_windows).  A candidate is an EPC record with
crc_ok == 1 (key = its bits) or else a slot whose fix is RECOVERED (key = the fix's bits).  It is rejected when
check_length is set and (key[0] >> 3) != 6, else when quality is given and the slot is EMPTY; every other candidate is
a read.  Tags are keyed by all 16 bytes and numbered by their first read in slot order.  Per tag: reads, recovered,
first / last slot, the peak read (largest p = f32(f64(re)^2 + f64(im)^2), ties to the lowest slot, NaN lowest), h of
the last read, first / last time = segs[s].offset + decim * (open_index + sync_index) in int64.
"""
import numpy as np

TAG_DTYPE = np.dtype([("epc", "u1", (16,)), ("reads", "<i4"), ("recovered", "<i4"), ("first_slot", "<i4"),
                      ("last_slot", "<i4"), ("peak_slot", "<i4"), ("peak_power", "<f4"), ("last_h_re", "<f4"),
                      ("last_h_im", "<f4"), ("first_time", "<i8"), ("last_time", "<i8")])
TAG_SUMMARY_DTYPE = np.dtype([("n_tags", "<i4"), ("reads", "<i4"), ("recovered", "<i4"), ("rejected_length", "<i4"),
                              ("rejected_empty", "<i4"), ("reserved", "<i4", (3,))])
NOT_CANDIDATE, REJECTED, NOT_STORED = -1, -2, -3   # read_tag codes (NOT_STORED: the slot is not written)
EPC, FIX_RECOVERED, SLOT_EMPTY = 1, 1, 0
NAN_BITS = 0x7fc00000


def power(h_re, h_im):
    """p = (float)((double)re*re + (double)im*im): both squares exact, the sum rounded in double, then to float"""
    x, y = np.asarray(h_re, dtype=np.float64), np.asarray(h_im, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (x * x + y * y).astype(np.float32)


def report(segs, recs, counts, quality=None, fixes=None, check_length=1, max_tags=1024, decim=5):
    """segs SEGMENT_DTYPE[nseg], recs RESULT_DTYPE[nseg, max_windows], counts int[nseg], quality QUALITY_DTYPE and fixes
    EPC_FIX_DTYPE shaped like recs (or None).  Returns (tags TAG_DTYPE[min(n_tags, max_tags)], summary
    TAG_SUMMARY_DTYPE record, read_tag int32[nseg * max_windows] with NOT_STORED where nothing is written)."""
    nseg, mw = recs.shape
    N = nseg * mw
    r = recs.reshape(-1)
    i = np.arange(N, dtype=np.int64)
    s = i // mw
    cnt = np.minimum(np.maximum(np.asarray(counts, dtype=np.int64), 0), mw)
    stored = (i % mw) < cnt[s] if N else np.zeros(0, dtype=bool)
    rec_ok = stored & (r["kind"] == EPC) & (r["crc_ok"] == 1)
    from_fix = np.zeros(N, dtype=bool)
    keys = r["bits"].copy()
    if fixes is not None:
        f = fixes.reshape(-1)
        from_fix = stored & ~rec_ok & (f["status"] == FIX_RECOVERED)
        keys[from_fix] = f["bits"][from_fix]
    cand = rec_ok | from_fix
    rej_len = cand & bool(check_length) & ((keys[:, 0] >> 3) != 6)
    rej_empty = np.zeros(N, dtype=bool)
    if quality is not None:
        rej_empty = cand & ~rej_len & (quality.reshape(-1)["outcome"] == SLOT_EMPTY)
    read = cand & ~rej_len & ~rej_empty
    read_tag = np.full(N, NOT_STORED, dtype=np.int32)
    read_tag[stored] = NOT_CANDIDATE
    read_tag[cand & ~read] = REJECTED

    idx = np.nonzero(read)[0]                       # ascending slots
    kv = np.ascontiguousarray(keys[idx]).view("V16").reshape(-1)
    if idx.size:
        _, first_pos, inv = np.unique(kv, return_index=True, return_inverse=True)
        inv = inv.reshape(-1)
    else:
        first_pos, inv = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    n_tags = first_pos.size
    number = np.empty(n_tags, dtype=np.int64)      # unique key -> tag index, by first read
    number[np.argsort(first_pos, kind="stable")] = np.arange(n_tags)
    tag = number[inv]
    read_tag[idx] = tag

    reads = np.bincount(tag, minlength=n_tags)
    recovered = np.bincount(tag, weights=from_fix[idx], minlength=n_tags).astype(np.int64)
    first = np.full(n_tags, np.iinfo(np.int64).max)
    np.minimum.at(first, tag, idx)
    last = np.full(n_tags, -1, dtype=np.int64)
    np.maximum.at(last, tag, idx)
    p = power(r["h_re"][idx], r["h_im"][idx])
    pk = np.where(np.isnan(p), np.uint64(0), p.view(np.uint32).astype(np.uint64) + np.uint64(1))
    comb = (pk << np.uint64(32)) | (~idx.astype(np.uint64) & np.uint64(0xFFFFFFFF))
    peak = np.zeros(n_tags, dtype=np.uint64)
    np.maximum.at(peak, tag, comb)

    def when(j):
        off = segs["offset"][j // mw].astype(np.uint64)
        d = (np.int64(decim) * (r["open_index"][j].astype(np.int64) + r["sync_index"][j].astype(np.int64)))
        return (off + d.astype(np.uint64)).view(np.int64)

    keep = min(n_tags, max_tags)
    out = np.zeros(keep, dtype=TAG_DTYPE)
    out["epc"] = keys[first[:keep]]
    out["reads"], out["recovered"] = reads[:keep], recovered[:keep]
    out["first_slot"], out["last_slot"] = first[:keep], last[:keep]
    pkk = (peak[:keep] >> np.uint64(32)).astype(np.uint32)
    out["peak_slot"] = (~peak[:keep]).astype(np.uint32).view(np.int32)   # the low word holds ~slot
    out["peak_power"] = np.where(pkk == 0, np.uint32(NAN_BITS), pkk - np.uint32(1)).astype(np.uint32).view(np.float32)
    out["last_h_re"], out["last_h_im"] = r["h_re"][last[:keep]], r["h_im"][last[:keep]]
    out["first_time"], out["last_time"] = when(first[:keep]), when(last[:keep])

    sm = np.zeros((), dtype=TAG_SUMMARY_DTYPE)
    sm["n_tags"], sm["reads"], sm["recovered"] = n_tags, idx.size, int(from_fix[idx].sum())
    sm["rejected_length"], sm["rejected_empty"] = int(rej_len.sum()), int(rej_empty.sum())
    return out, sm, read_tag
