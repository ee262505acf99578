"""GPU: tc_conv_kernel writes the same bits as the build that tests/golden/tc_conv_digests.json was recorded from.

A binarised network turns one flipped sign into a different run, so the forward / dgrad / eval kernel's results are
held bit for bit — dgrad output with every `add` arrangement and the fused BatchNorm statistics, both gradient
operand modes, every stride-2 phase, the int16 / fp32 / fp8 forward with its statistics, one eval unit per layer
shape, the stem — across changes to its main loop and epilogue.  Accuracy against fp64 is tests/test_gpu_tc.py's."""
import json
import os

import pytest

import tc_conv_digest_cases as C

pytestmark = pytest.mark.gpu

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tc_conv_digests.json")) as _fh:
    GOLDEN = json.load(_fh)


def test_fixture_covers_every_case():
    assert sorted(GOLDEN) == sorted(name for name, _ in C.all_cases())


@pytest.mark.parametrize("case", list(C.dgrad_cases()), ids=lambda c: c[0])
def test_dgrad_bits(case):
    assert C.run_dgrad(*case) == GOLDEN[case[0]]


@pytest.mark.parametrize("case", list(C.forward_cases()), ids=lambda c: c[0])
def test_forward_bits(case):
    assert C.run_forward(*case) == GOLDEN[case[0]]
