import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# Unit tests do not need the chain de-synchronisation pause (service.CONNECT_SLEEP_RANGE).
os.environ.setdefault("B200FED_CONNECT_SLEEP", "0,0")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `-m gpu`)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs")
