"""ctypes mirror of include/rfid_b200.h (structures and constants only).

Kept separate from the library loader so that test infrastructure can
share the record layout without importing the CUDA library.
"""
import ctypes as C

import numpy as np

RN16 = 0
EPC = 1
MAX_TAGS = 256

OK, EINVAL, ENODEV, ENOMEM, ECUDA, ECAPACITY = 0, -1, -2, -3, -4, -5


class Params(C.Structure):
    """rfid_b200_params (defaults: apps/reader.py:52-65, include/rfid/global_vars.h:72-143)."""
    _fields_ = [("adc_rate", C.c_int32), ("decim", C.c_int32), ("ntaps", C.c_int32),
                ("fixed_q", C.c_int32), ("max_queries", C.c_int32), ("max_tags", C.c_int32),
                ("device", C.c_int32), ("reserved", C.c_int32)]


class Segment(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("length", C.c_uint32), ("reserved", C.c_uint32)]


class WindowResult(C.Structure):
    _fields_ = [("segment", C.c_int32), ("window", C.c_int32), ("open_index", C.c_int32),
                ("length", C.c_int32), ("kind", C.c_int32), ("sync_index", C.c_int32),
                ("score", C.c_float), ("h_re", C.c_float), ("h_im", C.c_float), ("T", C.c_float),
                ("crc_ok", C.c_int32), ("tag_id", C.c_int32), ("bits", C.c_uint8 * 16)]


class Stats(C.Structure):
    _fields_ = [("n_queries_sent", C.c_int32), ("cur_inventory_round", C.c_int32),
                ("cur_slot_number", C.c_int32), ("max_slot_number", C.c_int32),
                ("n_epc_correct", C.c_int32), ("n_windows", C.c_int32), ("terminated", C.c_int32),
                ("n_unique_tags", C.c_int32), ("tag_id", C.c_int32 * MAX_TAGS),
                ("tag_reads", C.c_int32 * MAX_TAGS)]

    def tag_map(self):
        n = min(self.n_unique_tags, MAX_TAGS)
        return {int(self.tag_id[i]): int(self.tag_reads[i]) for i in range(n)}


class Segmenter(C.Structure):
    """rfid_b200_segmenter (include/rfid_b200.h): CW-gap segmenter settings."""
    _fields_ = [("level_frac", C.c_float), ("gap_us", C.c_float), ("lead_us", C.c_float),
                ("min_pulses", C.c_int32), ("commands_per_segment", C.c_int32), ("reserved", C.c_int32 * 3)]


class TxCommand(C.Structure):
    _fields_ = [("kind", C.c_int32), ("arg", C.c_int32)]


class SimParams(C.Structure):
    """rfid_b200_sim_params (include/rfid_b200.h): inventory-slot simulator settings."""
    _fields_ = [("seed", C.c_uint64), ("n_tags", C.c_int32), ("closed_loop", C.c_int32), ("dac_rate", C.c_int32),
                ("segment_us", C.c_float), ("lead_us", C.c_float), ("noise_sigma", C.c_float), ("tag_gain", C.c_float),
                ("tag_phase", C.c_float), ("clock_pct", C.c_float), ("leak_re", C.c_float), ("leak_im", C.c_float),
                ("floor_level", C.c_float), ("reserved", C.c_int32 * 2)]


TX_START, TX_QUERY, TX_QUERY_REP, TX_ACK, TX_CW, TX_NAK, TX_POWER_DOWN, TX_QUERY_ADJUST = range(8)
TX_COMMAND_DTYPE = np.dtype([("kind", "<i4"), ("arg", "<i4")])
SIM_TRUTH_DTYPE = np.dtype([("is_query", "<i4"), ("n_replies", "<i4"), ("strongest_rn16", "<i4"), ("acked_rn16", "<i4"),
                            ("replier", "<i4"), ("reserved", "<i4", (3,)), ("epc", "u1", (16,))])
assert C.sizeof(SimParams) == 64 and SIM_TRUTH_DTYPE.itemsize == 48 and C.sizeof(TxCommand) == 8
assert C.sizeof(Segmenter) == 32
assert C.sizeof(WindowResult) == 64
assert C.sizeof(Segment) == 16
assert C.sizeof(Params) == 32

#: numpy view of rfid_b200_window_result (same 64-byte layout)
RESULT_DTYPE = np.dtype([("segment", "<i4"), ("window", "<i4"), ("open_index", "<i4"), ("length", "<i4"),
                         ("kind", "<i4"), ("sync_index", "<i4"), ("score", "<f4"), ("h_re", "<f4"),
                         ("h_im", "<f4"), ("T", "<f4"), ("crc_ok", "<i4"), ("tag_id", "<i4"),
                         ("bits", "u1", (16,))])
SEGMENT_DTYPE = np.dtype([("offset", "<u8"), ("length", "<u4"), ("reserved", "<u4")])
assert RESULT_DTYPE.itemsize == 64 and SEGMENT_DTYPE.itemsize == 16

#: kind of a reader command that is none of Query, QueryRep, ACK, NAK, QueryAdjust (its bits are still stored)
CMD_OTHER = -1


class CmdParams(C.Structure):
    """rfid_b200_cmd_params (include/rfid_b200.h): reader-command decoder settings."""
    _fields_ = [("level_frac", C.c_float), ("level_abs", C.c_float), ("gap_us", C.c_float), ("reserved", C.c_int32 * 5)]


#: numpy view of rfid_b200_command (64 bytes)
COMMAND_DTYPE = np.dtype([("segment", "<i4"), ("index", "<i4"), ("start", "<i4"), ("end", "<i4"), ("kind", "<i4"),
                          ("n_bits", "<i4"), ("tari", "<i4"), ("rtcal", "<i4"), ("trcal", "<i4"), ("crc_ok", "<i4"),
                          ("arg", "<i4"), ("reserved", "<i4"), ("bits", "u1", (16,))])
assert COMMAND_DTYPE.itemsize == 64 and C.sizeof(CmdParams) == 32


SLOT_EMPTY, SLOT_SINGLE, SLOT_COLLISION = 0, 1, 2


class QualityParams(C.Structure):
    """rfid_b200_quality_params (include/rfid_b200.h): slot-outcome thresholds in dB."""
    _fields_ = [("empty_db", C.c_float), ("single_snr_db", C.c_float), ("reserved", C.c_int32 * 6)]


class Quality(C.Structure):
    _fields_ = [("energy", C.c_float), ("snr", C.c_float), ("outcome", C.c_int32), ("n_decisions", C.c_int32)]


#: numpy view of rfid_b200_quality (16 bytes): linear reply-energy and decision-SNR ratios, RFID_B200_SLOT_* outcome
QUALITY_DTYPE = np.dtype([("energy", "<f4"), ("snr", "<f4"), ("outcome", "<i4"), ("n_decisions", "<i4")])
assert QUALITY_DTYPE.itemsize == C.sizeof(Quality) == 16 and C.sizeof(QualityParams) == 32


FIX_CRC_OK, FIX_RECOVERED, FIX_AMBIGUOUS, FIX_FAILED, FIX_SKIPPED, FIX_NOT_EPC = range(6)


class RecoverParams(C.Structure):
    """rfid_b200_recover_params (include/rfid_b200.h): P least reliable positions, at most W flips, SNR gate in dB."""
    _fields_ = [("positions", C.c_int32), ("max_flips", C.c_int32), ("min_snr_db", C.c_float),
                ("reserved", C.c_int32 * 5)]


class EpcFix(C.Structure):
    _fields_ = [("status", C.c_int32), ("n_flips", C.c_int32), ("n_pass", C.c_int32), ("cost", C.c_float),
                ("bits", C.c_uint8 * 16)]


#: numpy view of rfid_b200_epc_fix (32 bytes): RFID_B200_FIX_* status, flips, passing candidates, cost, bits
EPC_FIX_DTYPE = np.dtype([("status", "<i4"), ("n_flips", "<i4"), ("n_pass", "<i4"), ("cost", "<f4"),
                          ("bits", "u1", (16,))])
assert EPC_FIX_DTYPE.itemsize == C.sizeof(EpcFix) == 32 and C.sizeof(RecoverParams) == 32


class ReportParams(C.Structure):
    """rfid_b200_report_params (include/rfid_b200.h): reject reads whose PC length field is not 6 words."""
    _fields_ = [("check_length", C.c_int32), ("reserved", C.c_int32 * 7)]


class Tag(C.Structure):
    _fields_ = [("epc", C.c_uint8 * 16), ("reads", C.c_int32), ("recovered", C.c_int32), ("first_slot", C.c_int32),
                ("last_slot", C.c_int32), ("peak_slot", C.c_int32), ("peak_power", C.c_float),
                ("last_h_re", C.c_float), ("last_h_im", C.c_float), ("first_time", C.c_int64),
                ("last_time", C.c_int64)]


class TagSummary(C.Structure):
    _fields_ = [("n_tags", C.c_int32), ("reads", C.c_int32), ("recovered", C.c_int32), ("rejected_length", C.c_int32),
                ("rejected_empty", C.c_int32), ("reserved", C.c_int32 * 3)]


#: numpy view of rfid_b200_tag (64 bytes): one tag of the inventory report
TAG_DTYPE = np.dtype([("epc", "u1", (16,)), ("reads", "<i4"), ("recovered", "<i4"), ("first_slot", "<i4"),
                      ("last_slot", "<i4"), ("peak_slot", "<i4"), ("peak_power", "<f4"), ("last_h_re", "<f4"),
                      ("last_h_im", "<f4"), ("first_time", "<i8"), ("last_time", "<i8")])
#: numpy view of rfid_b200_tag_summary (32 bytes)
TAG_SUMMARY_DTYPE = np.dtype([("n_tags", "<i4"), ("reads", "<i4"), ("recovered", "<i4"), ("rejected_length", "<i4"),
                              ("rejected_empty", "<i4"), ("reserved", "<i4", (3,))])
assert TAG_DTYPE.itemsize == C.sizeof(Tag) == 64 and TAG_SUMMARY_DTYPE.itemsize == C.sizeof(TagSummary) == 32
assert C.sizeof(ReportParams) == 32


MATCH_ALREADY_READ, MATCH_MATCHED, MATCH_AMBIGUOUS, MATCH_NO_MATCH, MATCH_SKIPPED, MATCH_NOT_EPC = range(6)
#: largest dictionary rfid_b200_match_epc accepts
MATCH_MAX_DICT = 1 << 24


class MatchParams(C.Structure):
    """rfid_b200_match_params (include/rfid_b200.h): largest cost and smallest margin, in mean reliabilities."""
    _fields_ = [("max_cost", C.c_float), ("min_margin", C.c_float), ("reserved", C.c_int32 * 6)]


class EpcMatch(C.Structure):
    _fields_ = [("status", C.c_int32), ("entry", C.c_int32), ("cost", C.c_int32), ("runner_up", C.c_int32),
                ("n_diff", C.c_int32), ("reserved", C.c_int32 * 3)]


class MatchCount(C.Structure):
    _fields_ = [("matched", C.c_int32), ("first_slot", C.c_int32), ("last_slot", C.c_int32), ("reserved", C.c_int32)]


#: numpy view of rfid_b200_epc_match (32 bytes): RFID_B200_MATCH_* status, entry, cost D1, runner-up D2, n_diff
EPC_MATCH_DTYPE = np.dtype([("status", "<i4"), ("entry", "<i4"), ("cost", "<i4"), ("runner_up", "<i4"),
                            ("n_diff", "<i4"), ("reserved", "<i4", (3,))])
#: numpy view of rfid_b200_match_count (16 bytes): one dictionary entry's MATCHED windows
MATCH_COUNT_DTYPE = np.dtype([("matched", "<i4"), ("first_slot", "<i4"), ("last_slot", "<i4"), ("reserved", "<i4")])
assert EPC_MATCH_DTYPE.itemsize == C.sizeof(EpcMatch) == 32 and MATCH_COUNT_DTYPE.itemsize == C.sizeof(MatchCount) == 16
assert C.sizeof(MatchParams) == 32


def make_segments(offsets, lengths):
    segs = np.zeros(len(offsets), dtype=SEGMENT_DTYPE)
    segs["offset"] = np.asarray(offsets, dtype=np.uint64)
    segs["length"] = np.asarray(lengths, dtype=np.uint32)
    return segs


def bits_hex(rec):
    """hex string of a record's decoded bits (4 hex digits for an RN16, 32 for an EPC)."""
    b = bytes(bytearray(rec["bits"]))
    return b[:2].hex() if int(rec["kind"]) == RN16 else b.hex()
