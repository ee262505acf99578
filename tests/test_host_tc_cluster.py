"""Host-only: the thread-block cluster the forward / dgrad planner picks for every network layer (no GPU)."""
import ctypes

LAYERS = [((64, 56, 56), 64, 1), ((64, 56, 56), 128, 2), ((128, 28, 28), 128, 1), ((128, 28, 28), 256, 2),
          ((256, 14, 14), 256, 1), ((256, 14, 14), 512, 2), ((512, 7, 7), 512, 1), ((64, 8, 8), 64, 1)]


def _plan(L, sh, mode, halves):
    out = (ctypes.c_int32 * 14)()
    assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), mode, halves, out, 14) == 0
    return list(out)


def test_cluster_choice_divides_the_grid_and_keeps_the_tiling(monkeypatch):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    L = _lib.lib()
    clustered = 0
    for n in (1, 2, 3, 256):
        for (cin, h, w), cout, stride in LAYERS:
            sh = conv_shape((n, cin, h, w), (cout, cin, 3, 3), stride, 1)
            for mode, halves in ((0, 1), (1, 1), (1, 2), (2, 1)):
                monkeypatch.setenv("BDBNN_TC_CLUSTER", "1")
                on = _plan(L, sh, mode, halves)
                monkeypatch.setenv("BDBNN_TC_CLUSTER", "0")
                off = _plan(L, sh, mode, halves)
                if not on[0]:
                    continue
                assert on[:12] == off[:12]                   # the per-CTA tiling does not depend on the cluster
                assert off[12:] == [1, 1]
                cm, cn = on[12:]
                BN, n_tiles, supers, grid = on[4], on[5], on[6], on[9]
                assert cm in (1, 2) and cn in (1, 2) and grid == supers * n_tiles
                assert supers % cm == 0 and n_tiles % cn == 0
                assert cm == (2 if supers % 2 == 0 else 1) and cn == (2 if n_tiles % 2 == 0 else 1)
                assert cn == 1 or BN * n_tiles >= 256            # N clusters only where there are two N tiles
                clustered += cm * cn > 1
    assert clustered > 60
