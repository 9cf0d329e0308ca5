import lzma
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def cfg1_iq():
    """The reference's recorded capture misc/data/file_source_test (committed xz-compressed)."""
    raw = lzma.decompress(open(os.path.join(GOLDEN, "file_source_test.c64.xz"), "rb").read())
    iq = np.frombuffer(raw, dtype=np.complex64)
    assert iq.size == 1247958
    return iq


@pytest.fixture(scope="session")
def cfg1_golden():
    return np.load(os.path.join(GOLDEN, "cfg1_ref_records.npy"))


@pytest.fixture(scope="session")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def ref_outputs():
    """What the reference's own blocks (oracle/_ref) computed on the inputs of the reference comparisons
    (tests/golden/make_golden.py: reference_outputs)."""
    with np.load(os.path.join(GOLDEN, "reference_outputs.npz")) as z:
        return {k: z[k] for k in z.files}


def records_equal(a, b):
    """bit-exact comparison of two record arrays; returns list of differing field names"""
    bad = []
    if a.shape != b.shape:
        return ["shape %s vs %s" % (a.shape, b.shape)]
    for f in a.dtype.names:
        if a[f].tobytes() != b[f].tobytes():
            bad.append(f)
    return bad
