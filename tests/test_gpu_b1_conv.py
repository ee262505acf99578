"""GPU: the binary tensor-core conv (csrc/b1_conv.cu, DESIGN.md §4x) — the bit order of one wgmma .b1.and.popc tile
against numpy, the exact int16 result against the 16-bit / fp8 wgmma kernel and the XNOR kernel, the eval epilogue's
z and sign words against the fp8 / 16-bit eval unit, and loaded 1-bit models whose logits stay bit-identical to the
source model's while their qualifying convs run on it."""
import ctypes

import numpy as np
import pytest
import torch

from b1_cases import B1_SHAPES, B1_MODEL_LAUNCHES, b1_shape_ok

pytestmark = pytest.mark.gpu


def _lib():
    from bdbnn_b200 import _lib as l
    return l


def _mma(a, b):
    from bdbnn_b200 import functional as F
    d = torch.empty((64, 8), dtype=torch.int32, device="cuda")
    A = torch.from_numpy(a.view(np.int32)).cuda()
    B = torch.from_numpy(b.view(np.int32)).cuda()
    _lib().check(_lib().lib().bdbnn_debug_b1_mma(F._p(A), F._p(B), F._p(d), F._stream()), "debug_b1_mma")
    return d.cpu().numpy()


def _mma_ref(a, b):
    x = np.unpackbits(a.view(np.uint8), bitorder="little").reshape(64, 256).astype(np.int64)
    y = np.unpackbits(b.view(np.uint8), bitorder="little").reshape(8, 256).astype(np.int64)
    return x @ y.T


def test_debug_b1_mma_random_bits():
    rng = np.random.default_rng(0)
    for _ in range(4):
        a = rng.integers(0, 2 ** 32, (64, 8), dtype=np.uint64).astype(np.uint32)
        b = rng.integers(0, 2 ** 32, (8, 8), dtype=np.uint64).astype(np.uint32)
        assert np.array_equal(_mma(a, b), _mma_ref(a, b))


def test_debug_b1_mma_single_bits():
    """bit j of word k is K element 32k + j: one set bit in A row m and B row n meets only itself."""
    for k in range(256):
        a = np.zeros((64, 8), dtype=np.uint32)
        b = np.zeros((8, 8), dtype=np.uint32)
        m, n = k % 64, k % 8
        a[m, k // 32] = np.uint32(1) << np.uint32(k % 32)
        b[n, k // 32] = np.uint32(1) << np.uint32(k % 32)
        b[(n + 1) % 8, ((k + 1) % 256) // 32] = np.uint32(1) << np.uint32((k + 1) % 32)   # a miss next to it
        want = np.zeros((64, 8), dtype=np.int64)
        want[m, n] = 1
        assert np.array_equal(_mma(a, b), want), k


def _inputs(n, cin, cout, hw, seed):
    """x with +-0.0 and NaN entries (act_pack: -0.0 -> +1, NaN -> -1), and +-1 weights (alpha = 1)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, hw, hw, generator=g)
    sel = torch.rand(x.shape, generator=g)
    x[sel < 0.02] = 0.0
    x[(sel >= 0.02) & (sel < 0.04)] = -0.0
    x[(sel >= 0.04) & (sel < 0.05)] = float("nan")
    w = torch.where(torch.rand(cout, cin, 3, 3, generator=g) < 0.5, -1.0, 1.0)
    return x.cuda().contiguous(memory_format=torch.channels_last), w.cuda()


def _packs(x, w, sh):
    from bdbnn_b200 import functional as F
    fmt = F.grad_mode()[3]
    ap = F._act_pack(x, sh, fmt, xb=True, xb8=bool(sh.Cin % 128 == 0))
    wp = F._alloc_weight_pack(w.shape, x.device, wf=True, wf8=sh.Cin % 128 == 0)
    F._weight_pack(w, wp, fmt)
    pw = F.PackedWeight(wp.wsign, wp.alpha, w.shape, {})
    return ap, wp, pw, fmt


def _b1_i16(ap, pw, sh):
    from bdbnn_b200 import functional as F
    y = torch.empty((sh.N, sh.Ho, sh.Wo, sh.Cout), dtype=torch.int16, device="cuda")
    _lib().check(_lib().lib().bdbnn_binconv_fwd_b1_i16(F._p(ap.sign), F._p(pw.sign), F._p(pw.popc_table()), F._p(y),
                                                      ctypes.byref(sh), F._stream()), "b1_i16")
    return y


@pytest.mark.parametrize("shape", B1_SHAPES)
def test_b1_i16_equals_wgmma_and_xnor(shape):
    from bdbnn_b200 import functional as F
    n, cin, cout, hw, stride = shape
    x, w = _inputs(n, cin, cout, hw, seed=cin + hw + stride)
    sh = F.conv_shape(x.shape, w.shape, stride, 1)
    caps = int(_lib().lib().bdbnn_tc_supported(ctypes.byref(sh)))
    assert caps & F.TC_B1 and b1_shape_ok(cin, cout, 3, stride, 1)
    ap, wp, pw, fmt = _packs(x, w, sh)
    assert torch.equal(wp.alpha, torch.ones_like(wp.alpha))
    y = _b1_i16(ap, pw, sh)
    y_xnor = F.binconv2d(x, w, stride, 1, "xnor")          # alpha * y_int with alpha = 1
    assert torch.equal(y.permute(0, 3, 1, 2).float(), y_xnor)
    if caps & 16:
        for use8 in ((False, True) if caps & 8 else (False,)):
            yt = torch.empty_like(y)
            F._fwd_tc(sh, use8, ap, wp, fmt, yt)
            assert torch.equal(y, yt), use8


def _eval_pair(x, w, sh, scale, shift, res):
    """(z, zbits) of the b1 eval kernel and z of the fp8 (16-bit when fp8 is not taken) eval kernel."""
    from bdbnn_b200 import functional as F
    L = _lib().lib()
    ap, wp, pw, fmt = _packs(x, w, sh)
    n_out = sh.N * sh.Ho * sh.Wo * sh.Cout
    z = torch.empty(n_out, device="cuda")
    zbits = torch.empty(n_out // 32, dtype=torch.int32, device="cuda")
    _lib().check(L.bdbnn_binconv_fwd_b1_eval(F._p(ap.sign), F._p(pw.sign), F._p(pw.popc_table()), F._p(scale),
                                             F._p(shift), F._p(res), F._p(z), F._p(zbits), ctypes.byref(sh),
                                             F._stream()), "b1_eval")
    use8 = sh.Cin % 128 == 0
    zt = torch.empty(n_out, device="cuda")
    _lib().check(L.bdbnn_binconv_fwd_tc_eval(F._p(ap.xb8 if use8 else ap.xb), F._p(wp.wf8 if use8 else wp.wf),
                                             -1 if use8 else fmt, F._p(scale), F._p(shift), F._p(res), F._p(zt), None,
                                             None, ctypes.byref(sh), F._stream()), "tc_eval")
    return z, zbits, zt


@pytest.mark.parametrize("residual", [None, "random", "zeros"])
@pytest.mark.parametrize("shape", [(2, 128, 128, 9, 1), (3, 256, 512, 7, 2), (1, 512, 512, 5, 1)])
def test_b1_eval_equals_eval_unit(shape, residual):
    from bdbnn_b200 import functional as F
    n, cin, cout, hw, stride = shape
    x, w = _inputs(n, cin, cout, hw, seed=7 + cin)
    g = torch.Generator().manual_seed(3)
    w = w * (torch.rand(cout, 1, 1, 1, generator=g).cuda() + 0.5)   # alpha != 1
    sh = F.conv_shape(x.shape, w.shape, stride, 1)
    gamma = torch.randn(cout, generator=g)
    beta = torch.randn(cout, generator=g)
    gamma[: cout // 8] = 0.0                       # channels with gamma = beta = 0: z = +-0.0
    beta[: cout // 8] = 0.0
    rm, rv = torch.randn(cout, generator=g), torch.rand(cout, generator=g) + 0.5
    alpha = w.abs().mean(dim=(1, 2, 3))
    scale, shift = F.bn_eval_fold(gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5, alpha)
    n_out = n * sh.Ho * sh.Wo * cout
    res = None
    if residual == "random":
        res = torch.randn(n_out, generator=g).cuda()
    elif residual == "zeros":                      # +0.0 and -0.0 residuals
        res = torch.where(torch.rand(n_out, generator=g) < 0.5, 0.0, -0.0).cuda()
    z, zbits, zt = _eval_pair(x, w, sh, scale, shift, res)
    assert torch.equal(z, zt)
    assert torch.equal(torch.signbit(z), torch.signbit(zt))
    zsh = F.conv_shape((n, cout, sh.Ho, sh.Wo), (cout, cout, 3, 3), 1, 1)
    ap = F._act_pack(z.view(n, sh.Ho, sh.Wo, cout).permute(0, 3, 1, 2), zsh, F.grad_mode()[3], xb=False, xb8=False)
    assert torch.equal(zbits, ap.sign.flatten())


def test_b1_refuses_other_shapes():
    from bdbnn_b200 import functional as F
    L = _lib().lib()
    d = torch.zeros(16, dtype=torch.int32, device="cuda")
    for xs, ws, stride, pad in (((1, 64, 8, 8), (64, 64, 3, 3), 1, 1), ((1, 384, 8, 8), (64, 384, 3, 3), 1, 1),
                                ((1, 128, 8, 8), (96, 128, 3, 3), 1, 1), ((1, 128, 8, 8), (64, 128, 1, 1), 1, 0)):
        sh = F.conv_shape(xs, ws, stride, pad)
        assert not int(L.bdbnn_tc_supported(ctypes.byref(sh))) & F.TC_B1
        rc = L.bdbnn_binconv_fwd_b1_i16(F._p(d), F._p(d), F._p(d), F._p(d), ctypes.byref(sh), F._stream())
        assert rc != 0


def _model_case(family, arch, monkeypatch, tmp_path):
    from bdbnn_b200 import export as E
    from test_gpu_export import _images, _source
    n, hw = (2, 224) if family == "imagenet" else (16, 32)
    src = _source(family, arch, n, hw)
    path = str(tmp_path / f"{arch}.bin")
    E.save_packed(src, path)
    return src, E.load_packed(path, "cuda"), _images(n, hw)


@pytest.mark.parametrize("family,arch", [("imagenet", "resnet18"), ("imagenet", "resnet34"), ("cifar", "resnet18"),
                                         ("cifar", "vgg_small"), ("cifar", "resnet20")])
def test_loaded_model_on_b1(family, arch, monkeypatch, tmp_path):
    from bdbnn_b200 import functional as F
    from bdbnn_b200.modules import PackedBinaryConv2d
    from test_gpu_export import _graphed
    monkeypatch.setenv("BDBNN_B1", "1")
    src, net, x = _model_case(family, arch, monkeypatch, tmp_path)
    with torch.no_grad():
        want = src(x)
        F.KernelTimer.start()
        got = net(x)
        rec = F.KernelTimer.stop()
    assert torch.equal(got, want)
    launches = {fam: sum(v["launches"] for (f, _), v in rec.items() if f == fam)
                for fam in ("binconv_fwd_b1_eval", "binconv_fwd_b1_i16")}
    assert launches == B1_MODEL_LAUNCHES[arch]
    for m in net.modules():
        if isinstance(m, PackedBinaryConv2d) and b1_shape_ok(m.in_channels, m.out_channels, m.kernel_size[0],
                                                             m.stride[0], m.padding[0]):
            assert set(m._operands) == {"b1"}          # no int16 or fp8 weight operand
    assert torch.equal(_graphed(net, x), want)
    monkeypatch.setenv("BDBNN_B1", "0")
    with torch.no_grad():
        F.KernelTimer.start()
        off = net(x)
        rec = F.KernelTimer.stop()
    assert torch.equal(off, want)
    assert not any(f.startswith("binconv_fwd_b1") for f, _ in rec)
