"""CPU: the arithmetic of the binary tensor-core conv (oracle/b1conv_ref.py, DESIGN.md §4x) against the integer conv
of oracle/binconv_ref.py, the popcount table, and which convs functional.use_b1 sends to the kernel."""
import numpy as np
import pytest
import torch

from b1_cases import B1_SHAPES, b1_shape_ok
from oracle import b1conv_ref as R
from oracle import binconv_ref as B


def _case(n, cin, cout, hw, signs, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, hw, hw, generator=g, dtype=torch.float64)
    w = torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64)
    if signs == "plus":
        x, w = x.abs(), w.abs()
    elif signs == "minus":
        x, w = -x.abs() - 1e-3, -w.abs() - 1e-3
    else:
        sel = torch.rand(x.shape, generator=g)
        x[sel < 0.05] = 0.0
        x[(sel >= 0.05) & (sel < 0.1)] = -0.0
        x[(sel >= 0.1) & (sel < 0.12)] = float("nan")
    return x, w


def _weight_words(w):
    """[Cout][9][Cin/32] sign words of an OIHW weight (bdbnn_weight_pack's wsign layout)."""
    cout, cin = w.shape[:2]
    t = w.numpy().reshape(cout, cin, 9, 1)      # NCHW with H = the 9 taps, W = 1
    return R.sign_words(t).reshape(cout, 9, -1)


@pytest.mark.parametrize("signs", ["random", "plus", "minus"])
@pytest.mark.parametrize("n,cin,cout,hw,stride", [(1, 128, 64, 5, 1), (2, 128, 64, 7, 2), (1, 256, 64, 6, 1),
                                                   (1, 256, 64, 5, 2), (1, 512, 64, 3, 1), (1, 512, 64, 4, 2),
                                                   (1, 128, 64, 1, 1), (1, 128, 64, 2, 2)])
def test_decomposition_equals_integer_conv(n, cin, cout, hw, stride, signs):
    x, w = _case(n, cin, cout, hw, signs, seed=cin + hw + stride)
    y = R.b1_conv_int(R.sign_words(x.numpy()), _weight_words(w), stride, cin)
    assert np.array_equal(y, B.binconv_int(x, w, stride, 1).numpy().astype(np.int64))


def test_paired_taps_at_cin_128():
    """At Cin = 128 a 256-bit K step holds two taps; the 9th tap is paired with a zero chunk in A and B."""
    x, w = _case(1, 128, 64, 4, "random", seed=1)
    xw, ww = R.sign_words(x.numpy()), _weight_words(w)
    a, b = R.k_chunks(xw, ww, 0, 1, 1, 1, 128)
    assert a.shape == (10, 4) and b.shape == (64, 10, 4)
    assert not a[9].any() and not b[:, 9].any()
    for t in range(9):
        ih, iw = t // 3, t % 3
        assert np.array_equal(a[t], xw[0, ih, iw]) and np.array_equal(b[:, t], ww[:, t])
    a, _ = R.k_chunks(xw, ww, 0, 0, 0, 1, 128)          # corner pixel: taps of row -1 and column -1 are zero
    for t in range(9):
        if t // 3 == 0 or t % 3 == 0:
            assert not a[t].any()
        else:
            assert np.array_equal(a[t], xw[0, t // 3 - 1, t % 3 - 1])


def test_popc_table():
    rng = np.random.default_rng(0)
    ww = rng.integers(0, 2 ** 32, (16, 9, 8), dtype=np.uint64).astype(np.uint32)
    table = R.popc_table(ww)
    want = np.array([[sum(bin(int(v)).count("1") for v in ww[o, t]) for t in range(9)] for o in range(16)])
    assert np.array_equal(table, want)
    assert np.array_equal(R.popc_table(np.full((2, 9, 4), 0xFFFFFFFF, dtype=np.uint32)), np.full((2, 9), 128))


def test_sign_words_of_zero_and_nan():
    x = np.array([0.0, -0.0, np.nan, 1.0, -1.0] + [1.0] * 27, dtype=np.float64).reshape(1, 32, 1, 1)
    assert int(R.sign_words(x)[0, 0, 0, 0]) & 0x1F == 0b01011


def _packed(cout, cin, k=3):
    from bdbnn_b200.functional import PackedWeight
    return PackedWeight(torch.zeros((cout, k * k, (cin + 31) // 32), dtype=torch.int32), torch.ones(cout),
                        (cout, cin, k, k), {})


def test_use_b1_selects_the_kernel_shapes(monkeypatch):
    from bdbnn_b200 import functional as F
    monkeypatch.setenv("BDBNN_B1", "1")
    for n, cin, cout, hw, stride in B1_SHAPES:
        sh = F.conv_shape((n, cin, hw, hw), (cout, cin, 3, 3), stride, 1)
        assert F.use_b1(sh, _packed(cout, cin)), (cin, cout, hw, stride)
        assert F.b1_selected(cin, cout, 3, stride, 1) == b1_shape_ok(cin, cout, 3, stride, 1)
    monkeypatch.setenv("BDBNN_B1", "0")
    sh = F.conv_shape((2, 128, 8, 8), (128, 128, 3, 3), 1, 1)
    assert not F.use_b1(sh, _packed(128, 128))


@pytest.mark.parametrize("cin,cout,k,stride,pad", [(64, 128, 3, 1, 1), (96, 128, 3, 1, 1), (384, 128, 3, 1, 1),
                                                    (1024, 128, 3, 1, 1), (128, 96, 3, 1, 1), (128, 128, 1, 1, 0),
                                                    (128, 128, 3, 1, 0)])
def test_use_b1_refusals(cin, cout, k, stride, pad, monkeypatch):
    from bdbnn_b200 import functional as F
    monkeypatch.setenv("BDBNN_B1", "1")
    sh = F.conv_shape((2, cin, 8, 8), (cout, cin, k, k), stride, pad)
    assert not F.use_b1(sh, _packed(cout, cin, k))


def test_use_b1_refuses_fp32_weights(monkeypatch):
    from bdbnn_b200 import functional as F
    monkeypatch.setenv("BDBNN_B1", "1")
    sh = F.conv_shape((2, 128, 8, 8), (128, 128, 3, 3), 1, 1)
    assert F.use_b1(sh, _packed(128, 128))
    assert not F.use_b1(sh, torch.zeros(128, 128, 3, 3))
