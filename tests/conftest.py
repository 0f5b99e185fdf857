import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    """tests/golden/<name>.npz, or the directory tests/golden/<name>/ of its parts (fixtures above 1 MB are split)."""
    from adanerf_b200.synthetic import load_npz
    p = os.path.join(GOLDEN, name)
    d = load_npz(p if os.path.isdir(p) else p + ".npz")
    d["meta"] = json.loads(str(d["meta"]))
    return d


def load_pavillon_weights():
    from adanerf_b200.synthetic import load_weights_npz
    return load_weights_npz(os.path.join(GOLDEN, "weights_pavillon"))


def case_weights(case):
    """Weights used to generate a golden stage case (see oracle/gen_golden.py)."""
    from oracle import adanerf_oracle as orc
    if case.startswith("pav"):
        return load_pavillon_weights()
    if case.startswith("shaped"):
        return orc.make_weights("shaped", seed=0)
    if case.startswith("ndc"):
        return orc.make_weights("ndc", seed=0)
    return orc.make_weights("rand", seed=0)


@pytest.fixture(scope="session")
def pavillon_weights():
    return load_pavillon_weights()
