"""CPU tests of the boundary: the C-ABI library builds, loads, exports every declared symbol, and refuses to
work without an H100 (no CPU fallback).  No compute calls here."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from gen2_uhf_rfid_reader_b200 import abi, capi


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "rfid_b200.h")).read()
    return sorted(set(re.findall(r"RFID_B200_API\s+[\w\s\*]+?\b(rfid_b200_\w+)\s*\(", hdr)))


def test_header_symbols_are_exported():
    lib = capi.load_library()
    names = _declared_symbols()
    assert len(names) >= 18
    assert sorted(names) == sorted(capi.EXPORTED_SYMBOLS)
    for n in names:
        assert hasattr(lib, n), n
    assert lib.rfid_b200_abi_version() == 1


def test_only_the_c_abi_is_exported():
    import subprocess
    out = subprocess.check_output(["nm", "-D", "--defined-only", capi.LIB], text=True)
    syms = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert syms and all(s.startswith("rfid_b200_") for s in syms), syms


def test_struct_layouts():
    assert C.sizeof(abi.WindowResult) == 64 and abi.RESULT_DTYPE.itemsize == 64
    assert C.sizeof(abi.Segment) == 16 and C.sizeof(abi.Params) == 32
    for name, _ in abi.WindowResult._fields_:
        if name != "bits":
            assert getattr(abi.WindowResult, name).offset == abi.RESULT_DTYPE.fields[name][1]
    assert abi.WindowResult.bits.offset == 48


def test_default_params_match_reference_constants():
    p = capi.default_params()
    # apps/reader.py:52-65, include/rfid/global_vars.h:72,76,100
    assert (p.adc_rate, p.decim, p.ntaps, p.fixed_q, p.max_queries, p.max_tags) == (2000000, 5, 25, 0, 1000, 100)


def test_error_strings():
    lib = capi.load_library()
    assert lib.rfid_b200_strerror(0) == b"ok"
    assert b"sm_90" in lib.rfid_b200_strerror(abi.ENODEV)
    assert lib.rfid_b200_strerror(-99) == b"unknown error"


def test_create_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(capi.RfidB200Error):
        capi.Gen2Rx()
    lib = capi.load_library()
    h = C.c_void_p()
    p = capi.default_params()
    assert lib.rfid_b200_create(C.byref(p), C.byref(h)) == abi.ENODEV and not h.value
    assert lib.rfid_b200_create(None, C.byref(h)) == abi.EINVAL
    bad = capi.default_params(decim=0)
    assert lib.rfid_b200_create(C.byref(bad), C.byref(h)) == abi.EINVAL


def test_sass_uses_tma_bulk_copy():
    """the fused kernel stages raw I/Q with cp.async.bulk (SASS UBLKCP) and waits on mbarriers"""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.check_output(["cuobjdump", "-sass", capi.LIB], text=True)
    assert "UBLKCP" in sass and "SYNCS.PHASECHK" in sass
    assert "sm_90a" in sass


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "gen2_uhf_rfid_reader_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("does not touch oracle/", "").lower(), os.path.join(dirpath, f)


def test_new_entry_points_reject_null_context_and_have_sane_defaults():
    """ingest / TX synthesiser / simulator entry points: argument checks come before any CUDA call"""
    lib = capi.load_library()
    n, ns = C.c_int(0), C.c_size_t(0)
    segs = np.zeros(4, dtype=abi.SEGMENT_DTYPE)
    x = np.zeros(8, dtype=np.float32)
    assert lib.rfid_b200_segment_capture(None, x.ctypes.data, 4, None, segs.ctypes.data, 4, C.byref(n), None) == abi.EINVAL
    assert lib.rfid_b200_ingest_capture_host(None, x.ctypes.data, 4, None, 2, segs.ctypes.data, 4, C.byref(n), None, None) == abi.EINVAL
    scr = np.zeros(1, dtype=abi.TX_COMMAND_DTYPE)
    assert lib.rfid_b200_tx_synth(None, scr.ctypes.data, 1, 1000000, None, 0, C.byref(ns), None) == abi.EINVAL
    sim = capi.default_sim()
    assert lib.rfid_b200_sim_segment_length(None, C.byref(sim)) == abi.EINVAL
    assert lib.rfid_b200_sim_capture(None, C.byref(sim), 0, 1, None, None, None, None) == abi.EINVAL
    # defaults: SURVEY 8d signal model, gate_impl.cc:164 pulse rule
    assert (sim.n_tags, sim.closed_loop, sim.dac_rate) == (1, 1, 1000000)
    assert abs(sim.segment_us - 8480.0) < 1e-3 and abs(sim.leak_re - 0.2846) < 1e-6 and abs(sim.noise_sigma - 0.003) < 1e-7
    sp = capi.default_segmenter()
    assert (sp.min_pulses, sp.commands_per_segment) == (6, 2) and sp.lead_us < sp.gap_us
    assert C.sizeof(abi.SimParams) == 64 and C.sizeof(abi.Segmenter) == 32 and abi.SIM_TRUTH_DTYPE.itemsize == 48


def test_sass_of_the_new_kernels_is_present():
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    out = subprocess.check_output(["cuobjdump", "-sass", capi.LIB], text=True)
    for k in ("ingest_mask", "ingest_scan", "ingest_bursts", "tx_synth_kernel", "sim_slot_kernel", "rx_fused_split_kernel", "rx_pack_kernel"):
        assert k in out, k


def test_create_refuses_rates_that_are_not_well_defined():
    """rfid_b200_create checks, before it looks for a device, that the reference decoder stays inside its windows at the
    configured rate (csrc/rfid_b200.cu: well_defined); against the independent numpy evaluation on the 1 kHz grid from
    1 to 8 MS/s: EINVAL exactly where the configuration is not well defined"""
    import rate_rule
    lib = capi.load_library()
    want = rate_rule.well_defined(rate_rule.GRID)
    h = C.c_void_p()
    rc = []
    for r in rate_rule.GRID:
        rc.append(lib.rfid_b200_create(C.byref(capi.default_params(adc_rate=int(r))), C.byref(h)))
        if rc[-1] == abi.OK:     # a GPU is present
            lib.rfid_b200_destroy(h)
    rc = np.array(rc)
    assert (rc[~want] == abi.EINVAL).all(), rate_rule.GRID[~want & (rc != abi.EINVAL)][:10]
    assert set(rc[want].tolist()) <= {abi.ENODEV, abi.OK}, rate_rule.GRID[want & (rc == abi.EINVAL)][:10]
    for adc in (1_520_000, 1_360_000, 5_800_000):
        with pytest.raises(capi.RfidB200Error, match="not well defined"):
            capi.Gen2Rx(adc_rate=adc)
