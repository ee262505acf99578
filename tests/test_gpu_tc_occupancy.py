"""Register and shared-memory budget of the forward / dgrad tensor-core kernel: the CUDA occupancy calculator must
allow two CTAs per SM at every ResNet-18 layer's tiling (a guard against, e.g., a dgrad instance growing back to 102
registers).  It checks what the calculator allows, not the residency reached at run time.

One CTA is 8 consumer warps; with one CTA per SM nothing overlaps a CTA's epilogue (the dgrad's loads of the added
shortcut gradient and of the STE mask) with another CTA's mainloop."""
import ctypes

import pytest

pytestmark = pytest.mark.gpu

LAYERS = [((64, 56, 56), 64, 1), ((64, 56, 56), 128, 2), ((128, 28, 28), 128, 1), ((128, 28, 28), 256, 2),
          ((256, 14, 14), 256, 1), ((256, 14, 14), 512, 2), ((512, 7, 7), 512, 1)]


@pytest.mark.parametrize("mode,halves", [(0, 1), (1, 1), (1, 2), (2, 1)])
def test_tc_conv_runs_two_ctas_per_sm_on_every_network_layer(mode, halves):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    L = _lib.lib()
    fmt = -1 if mode == 2 else (1 if halves == 2 else 0)        # fp8 / BDBNN_FMT_BF16 / BDBNN_FMT_FP16
    checked = 0
    for (cin, h, w), cout, stride in LAYERS:
        sh = conv_shape((256, cin, h, w), (cout, cin, 3, 3), stride, 1)
        plan = (ctypes.c_int32 * 12)()
        assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), mode, halves, plan, 12) == 0
        if not plan[0]:
            continue
        bn, smem = plan[4], plan[8]
        ctas = ctypes.c_int32(0)
        assert L.bdbnn_debug_tc_conv_ctas_per_sm(1 if mode == 1 else 0, fmt, bn, smem, ctypes.byref(ctas)) == 0
        assert ctas.value >= 2, ((cin, h, w), cout, stride, mode, halves, bn, smem, ctas.value)
        checked += 1
    assert checked >= 4


def test_ctas_per_sm_probe_rejects_bad_arguments():
    from bdbnn_b200 import _lib
    L = _lib.lib()
    ctas = ctypes.c_int32(0)
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(1, -1, 64, 0, ctypes.byref(ctas)) != 0     # fp8 is forward only
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(0, 0, 48, 0, ctypes.byref(ctas)) != 0      # no 48-column tile
