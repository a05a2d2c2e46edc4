import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests", "fake_comfy")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need an H100: on any other machine they are reported as skipped instead of failing in torch.cuda init."""
    import torch
    ok = torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    if ok:
        return
    why = pytest.mark.skip(reason="needs an H100 (sm_90) GPU")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(why)


@pytest.fixture(scope="session")
def pkg():
    import __graft_entry__ as ge
    ge.load_package()
    # A/B runs of kernel variants: GGUFB200_ALLOW_TUNING=1 GGUFB200_TEST_TUNING="key=value[,key=value]" runs the suite with
    # bench-only launch knobs set.
    for kv in filter(None, os.environ.get("GGUFB200_TEST_TUNING", "").split(",")):
        k, v = kv.split("=")
        assert ge._sub("_lib").lib().ggufb200_set_tuning(int(k), int(v)) == 0

    class NS:
        lib = ge._sub("_lib")
        dequant = ge._sub("dequant")
        ops = ge._sub("ops")
        loader = ge._sub("loader")
    return NS


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
