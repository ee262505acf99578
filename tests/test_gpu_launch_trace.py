"""GPU: the host layer asks the C ABI for the same calls as the version tests/golden/launch_trace.json.gz was recorded
from — the same entry points in the same order, with the same scalar and ConvShape arguments, the same NULL pointers,
the same launch counts and the same timed families, keys and bytes — for every workload and setting of
tests/launch_trace_cases.py.  What the results are is the other tests' business; this one holds the plumbing."""
import gzip
import json
import os

import pytest

import launch_trace_cases as C

pytestmark = pytest.mark.gpu

with gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "launch_trace.json.gz"), "rt") as _fh:
    GOLDEN = json.load(_fh)


def test_fixture_covers_every_case():
    assert sorted(GOLDEN) == sorted(f"{w}/{s}" for w in C.WORKLOADS for s in C.SETTINGS)


@pytest.mark.parametrize("setting", list(C.SETTINGS))
@pytest.mark.parametrize("workload", list(C.WORKLOADS))
def test_trace_equals_fixture(workload, setting):
    got = json.loads(json.dumps(C.trace(workload, setting)))      # tuples -> lists, as stored
    want = GOLDEN[f"{workload}/{setting}"]
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, f"event {i}: got {a}, recorded {b}"
    assert len(got) == len(want), f"{len(got)} events, {len(want)} recorded"
