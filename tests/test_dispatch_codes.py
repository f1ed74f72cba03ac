"""Every entry point of the dispatch layer returns the code tests/golden/dispatch_codes.json holds, for each of a few thousand
calls per entry point (tests/golden/make_dispatch_codes.py builds the calls): which check refuses an input, and which wins when
an input has several faults, is behaviour.  Without a CUDA device every call is refused, or fails at its launch, before any
kernel runs; with one, accepted calls would launch kernels on host buffers, so the test runs only where there is none."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_dispatch_codes as M  # noqa: E402


def _gpu_visible():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_gpu_visible(), reason="accepted calls would launch kernels on host buffers")
def test_every_entry_point_returns_the_golden_code_for_every_case():
    with open(M.GOLDEN) as f:
        golden = json.load(f)
    cases = M.cases()
    assert golden["cases"] == len(cases)
    L = M._lib.lib()
    n0 = L.fsr1_launch_count()
    codes = M.codes_of(L)
    assert L.fsr1_launch_count() == n0
    assert sorted(codes) == sorted(golden["codes"])
    for name in M.ENTRY_POINTS:
        got, want = codes[name], golden["codes"][name]
        assert len(got) == len(want) == len(cases)
        i = next((k for k in range(len(got)) if got[k] != want[k]), None)
        assert i is None, "%s returns %d instead of %d for case %d: %r" % (name, -int(got[i]), -int(want[i]), i, cases[i])
