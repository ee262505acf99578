"""The weight-gradient kernel in both operand modes (tc_wgrad.cu) against float64 conv2d_weight.

With +-1 activations, small-integer gradients (bf16, or fp16 with a power-of-two scale of 1), all-ones masks and unit
scales every product and every partial sum is an integer below 2^24, so the fp32 result is exact whatever the
summation order: gW must equal the float64 reference bit for bit.  In patch mode this checks that a row-shifted view
of a SWIZZLE_128B patch (a descriptor start 128 B * r * Wo into a 1024-byte-aligned tile) reads the rows TMA wrote
there."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

# (N, Cin, H, W, Cout, k, stride): every ResNet-18 binary conv at N = 7 and 256, then edge geometries
RESNET18 = [(64, 56, 64, 3, 1), (64, 56, 128, 3, 2), (128, 28, 128, 3, 1), (128, 28, 256, 3, 2),
            (256, 14, 256, 3, 1), (256, 14, 512, 3, 2), (512, 7, 512, 3, 1), (64, 28, 128, 1, 1), (256, 7, 512, 1, 1)]
GEOMS = [(n, c, hw, hw, co, k, s) for n in (7, 256) for c, hw, co, k, s in RESNET18] + [
    (1, 64, 56, 56, 64, 3, 1),        # one image
    (3, 64, 29, 29, 64, 3, 1),        # Ho prime: the last K stage of every image is partly outside it
    (2, 128, 23, 45, 64, 3, 1),       # rectangular, two patches per CTA
    (2, 64, 31, 31, 128, 3, 2),       # stride 2, odd size
    (1, 64, 20, 20, 64, 5, 1),        # 5x5 taps: views start up to 4 Wo rows into a patch
]


def _plan_mode(L, sh):
    out = (ctypes.c_int32 * 16)()
    assert L.bdbnn_debug_wgrad_plan(ctypes.byref(sh), 1, out, 16) == 0
    return out[12]


@pytest.mark.parametrize("mode", ["bf16", "fp16s"])
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "N{}_c{}_{}x{}_o{}_k{}s{}".format(*g))
def test_wgrad_tc_exact_for_integer_gradients(geom, mode):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import _p, _stream, conv_shape
    L = _lib.lib()
    n, cin, h, w, cout, k, stride = geom
    pad = k // 2
    sh = conv_shape((n, cin, h, w), (cout, cin, k, k), stride, pad)
    if k == 3 and stride == 1 and sh.Ho * sh.Wo > 128 and n == 256:
        assert _plan_mode(L, sh) == 1, geom
    g = torch.Generator(device="cuda").manual_seed(n + cin + h + cout + k)
    dev = torch.device("cuda")
    xb = torch.where(torch.rand(n, h, w, cin, device=dev, generator=g) < 0.5, -1.0, 1.0)
    gy = torch.randint(-4, 5, (n, sh.Ho, sh.Wo, cout), device=dev, generator=g).float()
    # fp16s: max|g| = 2^13 gives the power-of-two scale 1 (amax_pow2_scale), so gys holds the integers themselves
    dt, code = (torch.bfloat16, 1) if mode == "bf16" else (torch.float16, 3)
    amax = torch.tensor([0x46000000], dtype=torch.int32, device=dev) if code == 3 else None
    xb16 = xb.to(dt).view(torch.int16).contiguous()
    gy16 = gy.to(dt).view(torch.int16).contiguous()
    nw = cout * cin * k * k
    wmask = torch.full(((nw + 31) // 32,), -1, dtype=torch.int32, device=dev)
    inv_gscale = torch.ones(cout, device=dev)
    gw = torch.full((cout, cin, k, k), float("nan"), device=dev)
    nbytes = int(L.bdbnn_wgrad_tc_workspace_bytes(ctypes.byref(sh)))
    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
    _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gy16), code, _p(amax), _p(xb16), _p(wmask), _p(inv_gscale), _p(gw),
                                        ctypes.byref(sh), _p(ws), nbytes, _stream()), "binconv_wgrad_tc")
    ref = torch.nn.grad.conv2d_weight(xb.permute(0, 3, 1, 2).double(), (cout, cin, k, k),
                                      gy.permute(0, 3, 1, 2).double(), stride=stride, padding=pad)
    got = gw.double()
    bad = (got != ref).sum().item()
    assert bad == 0, (geom, bad, (got - ref).abs().max().item())


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
def test_wgrad_patch_mode_error_vs_fp64_layer2(mode, monkeypatch):
    """The 28x28 stride-1 layer at N = 256 (patch mode, two patches per CTA) with a heavy-tailed real gradient:
    the weight gradient stays within the mode's tolerances against float64 (as the full-size tests of the other
    layers do)."""
    from bdbnn_b200.functional import binconv2d
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    g = torch.Generator(device="cuda").manual_seed(261)
    x = (torch.randn(256, 128, 28, 28, device="cuda", generator=g) * 1.2).contiguous(memory_format=torch.channels_last)
    w = torch.randn(128, 128, 3, 3, device="cuda", generator=g) * 0.6
    wd = w.clone().requires_grad_(True)
    y = binconv2d(x, wd, 1, 1, "tc")
    gy = torch.randn(y.shape, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    gy = gy * torch.exp(2.0 * torch.randn(y.shape[0], 1, 1, 1, device="cuda", generator=g)) * 1e-3
    y.backward(gy)
    xb = torch.where(x >= 0, 1.0, -1.0).double()
    ref = torch.nn.grad.conv2d_weight(xb, w.shape, gy.double(), stride=1, padding=1) * (w.abs() <= 1)
    err = wd.grad.double() - ref
    e_max = err.abs().max().item() / ref.abs().max().item()
    e_l2 = err.norm().item() / ref.norm().item()
    assert e_max <= {"fp16s": 1.5e-3, "bf16x2": 5e-5}[mode], e_max
    assert e_l2 <= {"fp16s": 1e-3, "bf16x2": 2e-5}[mode], e_l2
