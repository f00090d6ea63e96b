import pathlib
import sys

import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) device")


@pytest.fixture(scope="session")
def oa():
    import oracle_api
    oracle_api.lib()
    return oracle_api


@pytest.fixture(scope="session")
def api():
    import multicol_slam_b200.api as a
    a.lib()
    return a


@pytest.fixture(scope="session")
def cams():
    from multicol_slam_b200 import synth
    return synth.lafida_cams()
