import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine with one)")


def has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def oracle():
    import lcs_oracle
    lcs_oracle.lib()
    return lcs_oracle


@pytest.fixture(scope="session")
def lcs():
    import lcs_b200
    lcs_b200.build()
    lcs_b200.lib()
    return lcs_b200


@pytest.fixture(scope="session")
def ctx(lcs):
    if not has_gpu():
        pytest.skip("no GPU")
    c = lcs.Context(0)
    yield c
    c.close()


def load(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.fixture(scope="session")
def capbuf0000():
    g = load("capbuf_0000.npz")
    cu8 = g["cu8"].reshape(-1, 2)
    cap = ((cu8.astype(np.float64) - 127) / 128).view(np.complex128).reshape(-1)
    return dict(cu8=cu8, capbuf=cap, fc=float(g["fc"][0]))


def synth_cu8(seed, n_cap=153600, sigma=20.0):
    """rtl-sdr-like 8-bit IQ (SURVEY 8d config 2): clip(round(127.5 + sigma*N(0,1)), 0, 255)."""
    rng = np.random.default_rng(seed)
    v = np.clip(np.round(127.5 + sigma * rng.standard_normal((n_cap, 2))), 0, 255)
    return v.astype(np.uint8)


def cu8_to_c128(cu8):
    return ((cu8.astype(np.float64) - 127) / 128).view(np.complex128).reshape(-1)
