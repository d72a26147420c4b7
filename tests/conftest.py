import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def golden_cases():
    import json
    out = []
    for name in sorted(os.listdir(GOLDEN)):
        gj = os.path.join(GOLDEN, name, "golden.json")
        if os.path.exists(gj):
            g = json.load(open(gj))
            for k, v in sorted(g["by_k"].items(), key=lambda kv: int(kv[0])):
                out.append(pytest.param(name, int(k), g["m"], v, id=f"{name}-k{k}"))
    return out
