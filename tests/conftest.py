import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py


@pytest.fixture(scope="session")
def oracle_blend():
    """the oracle compiled with the reference's feature="blend" probability model (oracle/oracle_blend.py)"""
    from oracle import oracle_blend as ob
    ob.build()
    return ob


@pytest.fixture(scope="session")
def golden():
    import json
    d = os.path.join(ROOT, "tests", "golden")
    idx = json.load(open(os.path.join(d, "golden.json")))
    for e in idx:
        e["path"] = os.path.join(d, e["name"] + ".divans")
    return idx


@pytest.fixture(scope="session")
def engine():
    import divans_b200
    eng = divans_b200.Engine(0, 0, int(os.environ.get("DIVANS_B200_LPS", "16")))   # default: the v2 engine, two streams per warp
    yield eng
    eng.close()


@pytest.fixture(scope="session")
def engine16():
    # the other lane layout of the v2 engine: four streams per warp, two CDF elements per lane
    import divans_b200
    eng = divans_b200.Engine(0, 64, 8)
    yield eng
    eng.close()


@pytest.fixture(scope="session")
def engine32():
    import divans_b200
    eng = divans_b200.Engine(0, 64, 32)
    yield eng
    eng.close()
