import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (runs under `pytest -m gpu`)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    return np.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))


def pytest_report_header(config):
    """Which GPU ran the `-m gpu` tests (serial number, clocks, ECC state): GPUs of a pool differ, and a mismatch
    that never reproduces can only be followed up with this."""
    import shutil
    import subprocess

    if shutil.which("nvidia-smi") is None:
        return None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,serial,uuid,vbios_version,clocks.sm,clocks.max.sm,"
                              "temperature.gpu,ecc.errors.uncorrected.volatile.total", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return None
    return [f"gpu: {line}" for line in out.splitlines()] or None
