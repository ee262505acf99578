"""GPU: the forward / dgrad tensor-core kernel with thread-block clusters (TMA multicast of the weight and activation
boxes that neighbouring CTAs share, BDBNN_TC_CLUSTER=1) computes bit-identical results to one-CTA launches.

Operands are random bit patterns of the right formats; what is checked is that the cluster launch changes nothing,
including the fixed-order BatchNorm statistics.  Correctness against the fp64 oracle is tests/test_gpu_tc.py's."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

# n, cin, h, w, cout, stride: the ResNet-18 3x3 layers at small N, plus grids with an odd M tile count (cluster
# falls back to one CTA along M)
SHAPES = [(2, 64, 56, 56, 64, 1), (2, 64, 56, 56, 128, 2), (2, 128, 28, 28, 128, 1), (2, 128, 28, 28, 256, 2),
          (2, 256, 14, 14, 256, 1), (2, 256, 14, 14, 512, 2), (2, 512, 7, 7, 512, 1),
          (1, 512, 7, 7, 512, 1), (3, 128, 28, 28, 128, 1)]
FP16_ONE, FP16_MINUS_ONE = 0x3C00, 0xBC00
FP8_ONE, FP8_MINUS_ONE = 0x38, 0xB8


def _lib():
    from bdbnn_b200 import _lib as lb
    return lb.lib()


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _shape(n, cin, h, w, cout, stride):
    from bdbnn_b200.functional import conv_shape
    return conv_shape((n, cin, h, w), (cout, cin, 3, 3), stride, 1)


def _pm1(g, numel, one, minus_one, dtype):
    bits = torch.randint(0, 2, (numel,), generator=g, dtype=torch.int32)
    return torch.where(bits == 1, one, minus_one).to(dtype).cuda()


def _both(monkeypatch, run):
    """run() with clusters off, then on; returns both results (tuples of tensors)."""
    out = []
    for flag in ("0", "1"):
        monkeypatch.setenv("BDBNN_TC_CLUSTER", flag)
        out.append(run())
        torch.cuda.synchronize()
    return out


def _assert_same(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


def test_plan_probe_reports_clusters_and_the_switch(monkeypatch):
    L = _lib()
    sh = _shape(2, 256, 14, 14, 256, 1)
    out = (ctypes.c_int32 * 14)()
    monkeypatch.setenv("BDBNN_TC_CLUSTER", "1")
    assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), 1, 1, out, 14) == 0
    assert (out[12], out[13]) == (2, 2)
    monkeypatch.setenv("BDBNN_TC_CLUSTER", "0")
    assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), 1, 1, out, 14) == 0
    assert (out[12], out[13]) == (1, 1)


@pytest.mark.parametrize("add_mode", ["none", "separate", "in_place", "stats"])
@pytest.mark.parametrize("shape", SHAPES)
def test_dgrad_cluster_bit_identical(shape, add_mode, monkeypatch):
    n, cin, h, w, cout, stride = shape
    if add_mode == "stats" and stride != 1:
        pytest.skip("the fused statistics need stride 1")
    L = _lib()
    sh = _shape(*shape)
    ho, wo = sh.Ho, sh.Wo
    g = torch.Generator().manual_seed(hash(shape) % 1000 + len(add_mode))
    gys = (torch.randn(n * ho * wo * cout, generator=g) * 0.5).half().cuda().view(torch.int16)
    wt = _pm1(g, cin * 9 * cout, FP16_ONE, FP16_MINUS_ONE, torch.int16)
    amax = torch.tensor([4.0]).view(torch.int32).cuda()
    npx = n * h * w
    mask = torch.randint(-2**31, 2**31 - 1, (npx * ((cin + 31) // 32),), generator=g, dtype=torch.int64)
    mask = mask.to(torch.int32).cuda()
    add0 = torch.randn(npx * cin, generator=g).cuda()
    y_int = torch.randint(-300, 300, (npx * cin,), generator=g, dtype=torch.int16).cuda()
    st_a, st_m = (torch.rand(cin, generator=g) + 0.5).cuda(), torch.randn(cin, generator=g).cuda()
    st_i = (torch.rand(cin, generator=g) + 0.5).cuda()

    def run():
        gx = torch.full((npx * cin,), 7.0, device="cuda")
        add = None
        if add_mode in ("separate", "stats"):
            add = add0.clone()
        elif add_mode == "in_place":
            gx.copy_(add0)
            add = gx
        if add_mode == "stats":
            sums = torch.zeros(2 * cin, dtype=torch.float64, device="cuda")
            gmax = torch.zeros(cin, dtype=torch.int32, device="cuda")
            assert L.bdbnn_binconv_dgrad_tc_stats(_p(gys), 3, _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                                  ctypes.byref(sh), _p(y_int), _p(st_a), _p(st_m), _p(st_i),
                                                  _p(sums), _p(gmax), _stream()) == 0
            return gx, sums, gmax
        assert L.bdbnn_binconv_dgrad_tc(_p(gys), 3, _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                        ctypes.byref(sh), _stream()) == 0
        return (gx,)

    off, on = _both(monkeypatch, run)
    _assert_same(off, on)


@pytest.mark.parametrize("kind", ["fp16", "fp8", "i16"])
@pytest.mark.parametrize("shape", SHAPES)
def test_forward_cluster_bit_identical(shape, kind, monkeypatch):
    n, cin, h, w, cout, stride = shape
    if kind == "fp8" and cin % 128 != 0:
        pytest.skip("the fp8 forward needs Cin % 128 == 0")
    L = _lib()
    sh = _shape(*shape)
    g = torch.Generator().manual_seed(hash(shape) % 1000 + len(kind))
    if kind == "fp8":
        xb = _pm1(g, n * h * w * cin, FP8_ONE, FP8_MINUS_ONE, torch.uint8)
        wf = _pm1(g, cout * 9 * cin, FP8_ONE, FP8_MINUS_ONE, torch.uint8)
    else:
        xb = _pm1(g, n * h * w * cin, FP16_ONE, FP16_MINUS_ONE, torch.int16)
        wf = _pm1(g, cout * 9 * cin, FP16_ONE, FP16_MINUS_ONE, torch.int16)
    alpha = (torch.rand(cout, generator=g) + 0.1).cuda()
    npo = n * sh.Ho * sh.Wo

    def run():
        sums = torch.zeros(2 * cout, dtype=torch.float64, device="cuda")
        ymax = torch.zeros(cout, dtype=torch.int32, device="cuda")
        if kind == "i16":
            y = torch.zeros(npo * cout, dtype=torch.int16, device="cuda")
            rc = L.bdbnn_binconv_fwd_tc_i16(_p(xb), _p(wf), 0, _p(alpha), _p(y), ctypes.byref(sh), _p(sums),
                                            _p(ymax), _stream())
        elif kind == "fp8":
            y = torch.zeros(npo * cout, device="cuda")
            rc = L.bdbnn_binconv_fwd_tc8(_p(xb), _p(wf), _p(alpha), _p(y), ctypes.byref(sh), _p(sums), _p(ymax),
                                         _stream())
        else:
            y = torch.zeros(npo * cout, device="cuda")
            rc = L.bdbnn_binconv_fwd_tc(_p(xb), _p(wf), 0, _p(alpha), _p(y), ctypes.byref(sh), _p(sums), _p(ymax),
                                        _stream())
        assert rc == 0
        return y, sums, ymax

    off, on = _both(monkeypatch, run)
    _assert_same(off, on)


@pytest.mark.parametrize("n,h,w", [(2, 224, 224), (1, 64, 64), (3, 33, 47)])
def test_stem_cluster_bit_identical(n, h, w, monkeypatch):
    L = _lib()
    assert L.bdbnn_stem_supported(n, h, w)
    g = torch.Generator().manual_seed(n * h + w)
    x = torch.randn(n, 3, h, w, generator=g).cuda()
    weight = torch.randn(64, 3, 7, 7, generator=g).cuda()
    xw = torch.zeros(int(L.bdbnn_stem_xw_bytes(n, h, w)), dtype=torch.uint8, device="cuda")
    x_amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    wf = torch.zeros(64 * 7 * 32, dtype=torch.int16, device="cuda")
    alpha = torch.zeros(64, device="cuda")
    st = x.stride()
    assert L.bdbnn_stem_pack(_p(x), n, h, w, st[0], st[1], st[2], st[3], _p(weight), _p(xw), _p(x_amax), _p(wf),
                             _p(alpha), _stream()) == 0
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1

    def run():
        y = torch.zeros(n * ho * wo * 64, device="cuda")
        sums = torch.zeros(128, dtype=torch.float64, device="cuda")
        ymax = torch.zeros(64, dtype=torch.int32, device="cuda")
        assert L.bdbnn_stem_conv_fwd(_p(xw), _p(wf), _p(alpha), _p(y), n, h, w, _p(sums), _p(ymax), _stream()) == 0
        return y, sums, ymax

    off, on = _both(monkeypatch, run)
    _assert_same(off, on)
