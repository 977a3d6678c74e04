import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def golden(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


def csr_from_coo(coo_u, coo_i, user_num):
    """user->item CSR with sorted unique columns (set semantics of get_ur, daisy/utils/utils.py:19-34)."""
    key = np.unique(coo_u.astype(np.int64) * (1 << 32) + coo_i.astype(np.int64))
    u = (key >> 32).astype(np.int64)
    col = (key & 0xFFFFFFFF).astype(np.int32)
    row_ptr = np.zeros(user_num + 1, np.int64)
    np.add.at(row_ptr, u + 1, 1)
    return np.cumsum(row_ptr), col
