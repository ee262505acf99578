"""Register budget of the binary tensor-core conv (csrc/b1_conv.cu, DESIGN.md §4x), read from the ptxas report the
build keeps (bdbnn_b200/build/nvcc.log, -Xptxas -v): no instance spills, and each stays within 96 registers, so that
two 256-thread CTAs fit an SM's 65 536 registers (at Cin = 512 their 110.6 KB of shared memory allow two as well)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "bdbnn_b200", "build", "nvcc.log")


def _b1_entries():
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    text = open(LOG).read().split("== b1_conv.cu", 1)
    assert len(text) == 2, "b1_conv.cu is not in the build"
    body = text[1].split("\n== ", 1)[0]
    out = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
                         r"ptxas info\s*: Used (\d+) registers", body, re.S):
        out[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
    return out


def test_b1_conv_instances_fit_two_ctas_per_sm_without_spills():
    entries = {k: v for k, v in _b1_entries().items() if "b1_conv_kernel" in k}
    assert len(entries) == 6                               # eval / int16 x Cin 128, 256, 512
    for name, (st, ld, regs) in entries.items():
        assert st == 0 and ld == 0, name
        assert regs <= 96, (name, regs)
