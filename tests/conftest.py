import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu, exclude with -m 'not gpu'")


@pytest.fixture(scope="session")
def oracle():
    from oracle.pinot_oracle import oracle as get
    return get()


@pytest.fixture(scope="session")
def sv_columns():
    """The 11 columns of the reference's test_data-sv.avro fixture (tests/golden/make_golden.py)."""
    d = np.load(os.path.join(ROOT, "tests", "golden", "test_data_sv.npz"))
    return {k: d[k] for k in d.files}


SV_INVERTED = ["column6", "column7", "column11", "column17", "column18"]  # BaseSingleValueQueriesTest.java:94


@pytest.fixture(scope="session")
def sv_segment(oracle, sv_columns):
    """Pinot-format index buffers of the reference's single-value test segment."""
    return oracle.build_segment("testTable_126164076_167572854", sv_columns, inverted=SV_INVERTED)
