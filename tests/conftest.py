import json
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real CUDA device (an sm_90a GPU: H100)")


@pytest.fixture(scope="session")
def golden():
    with open(ROOT / "tests" / "golden" / "reference_asserts.json") as f:
        return json.load(f)
