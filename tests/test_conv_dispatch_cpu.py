"""The engine's convolution dispatch on the CPU: for each network, precision setting and convolution switch, the native
launches of one forward (and backward) step -- which kernel every convolution runs on, its operand forms, statistics,
scales and the launch order -- against tests/golden/dispatch_trace.json.gz (see tests/golden/make_dispatch_trace.py)."""
import importlib.util
import json
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "make_dispatch_trace", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_dispatch_trace.py"))
T = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(T)


@pytest.fixture(scope="module")
def golden():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native
    if _native.lib().fpd_sm_count() != T.SM_COUNT:
        pytest.skip("the trace is recorded for %d SMs" % T.SM_COUNT)
    return T.load()


def test_fixture_holds_every_case_and_is_canonical(golden):
    assert sorted(golden) == sorted(T.CASES)
    with open(T.OUT, "rb") as f:
        assert T.dumps(golden) == f.read()


@pytest.mark.parametrize("case", T.CASES)
def test_launches_match_the_recorded_trace(case, golden):
    got = json.loads(json.dumps(T.trace(case)))
    want = golden[case]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (case, i)
    assert len(got) == len(want), case
