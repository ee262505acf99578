"""GPU parity tests: every kernel is called through the C ABI (ctypes) and compared with the CPU
oracle on the same seeded inputs.  Bit-exact for sign/pack and the integer part of the forward;
stated fp32 tolerances elsewhere."""
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import binconv_ref as B      # noqa: E402
from oracle import losses_ref as Lr      # noqa: E402


def _env():
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import _p, _stream, conv_shape
    return _lib, _lib.lib(), _p, _stream, conv_shape


def _u32(words):           # oracle int64 words -> comparable int64 from int32 device tensors
    return words


def _as_u32(t):
    return t.cpu().to(torch.int64) & 0xFFFFFFFF


def _nhwc(x):
    return x.cuda().contiguous(memory_format=torch.channels_last)


PACK_SHAPES = [(2, 64, 7, 5), (1, 3, 4, 4), (3, 16, 5, 6), (2, 40, 3, 9), (1, 100, 2, 2),
               (1, 128, 9, 1), (4, 32, 1, 1), (2, 512, 7, 7)]


@pytest.mark.parametrize("shape", PACK_SHAPES)
@pytest.mark.parametrize("with_bf16", [False, True])
def test_act_pack_bit_exact(shape, with_bf16):
    _lib, L, _p, _stream, _ = _env()
    n, c, h, w = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g) * 1.3
    flat = x.view(-1)
    flat[0], flat[1], flat[2], flat[3] = 0.0, -0.0, 1.0, -1.0
    if flat.numel() > 8:
        flat[4], flat[5], flat[6], flat[7] = float("nan"), float("inf"), -float("inf"), 1.0000001
    xc = _nhwc(x)
    cw = (c + 31) // 32
    sb = torch.full((n, h, w, cw), -1, dtype=torch.int32, device="cuda")
    mb = torch.full((n, h, w, cw), -1, dtype=torch.int32, device="cuda")
    fmt = 1 if sum(shape) % 2 else 0            # alternate bf16 / fp16 encodings of +-1
    xdt = torch.bfloat16 if fmt == 1 else torch.float16
    xb = torch.zeros((n, h, w, c), dtype=xdt, device="cuda") if with_bf16 else None
    _lib.check(L.bdbnn_act_pack(_p(xc), n * h * w, c, _p(sb), _p(mb), _p(xb), fmt, _stream()), "act_pack")
    torch.cuda.synchronize()
    assert torch.equal(_as_u32(sb), B.pack_bits_nhwc(x))
    assert torch.equal(_as_u32(mb), B.pack_mask_nhwc(x))
    if with_bf16:
        assert torch.equal(xb.float().cpu(), B.sign_pm1(x).permute(0, 2, 3, 1))


def test_act_pack_empty_is_ok():
    _lib, L, _p, _stream, _ = _env()
    e = torch.empty(0, device="cuda")
    assert L.bdbnn_act_pack(_p(e), 0, 64, _p(e), _p(e), _p(None), 1, _stream()) == 0


def test_bad_arguments_return_error_codes():
    _lib, L, _p, _stream, conv_shape = _env()
    e = torch.empty(4, device="cuda")
    assert L.bdbnn_act_pack(_p(e), 4, 0, _p(e), _p(e), _p(None), 1, _stream()) == -1
    assert L.bdbnn_act_pack(_p(e), 4, 32, _p(e), _p(e), _p(None), 7, _stream()) == -1
    assert b"act_pack" in L.bdbnn_last_error_string()
    sh = conv_shape((1, 4, 5, 5), (4, 4, 3, 3), 1, 1)
    sh.Ho = 7
    assert L.bdbnn_binconv_fwd_xnor(_p(e), _p(e), _p(e), _p(e), ctypes.byref(sh), _stream()) == -1
    with pytest.raises(RuntimeError, match="failed with code"):
        _lib.check(-1, "demo")


WSHAPES = [(64, 64, 3, 3), (5, 3, 3, 3), (16, 16, 3, 3), (8, 40, 1, 1), (128, 64, 1, 1), (4, 33, 5, 5)]


@pytest.mark.parametrize("shape", WSHAPES)
def test_weight_pack(shape):
    _lib, L, _p, _stream, _ = _env()
    cout, cin, kh, kw = shape
    T, cw = kh * kw, (cin + 31) // 32
    g = torch.Generator().manual_seed(11 + sum(shape))
    wt = torch.randn(shape, generator=g) * 0.7
    wt.view(-1)[0] = 0.0
    wt.view(-1)[1] = 1.0
    wt.view(-1)[2] = -1.0000001
    if cout > 1:
        wt[1].zero_()                       # alpha == 0 filter: sign(0)=+1, gscale=1, wt operand zeroed
    wd = wt.cuda()
    alpha = torch.empty(cout, device="cuda")
    ws = torch.empty((cout, T, cw), dtype=torch.int32, device="cuda")
    wm = torch.empty(((wt.numel() + 31) // 32,), dtype=torch.int32, device="cuda")
    fmt = 1 if sum(shape) % 2 else 0
    wdt = torch.bfloat16 if fmt == 1 else torch.float16
    wf = torch.empty((cout, T, cin), dtype=wdt, device="cuda")
    wtt = torch.empty((cin, T, cout), dtype=wdt, device="cuda")
    gs = torch.empty(cout, device="cuda")
    igs = torch.empty(cout, device="cuda")
    wf8 = torch.zeros((cout, T, cin), dtype=torch.uint8, device="cuda")
    _lib.check(L.bdbnn_weight_pack(_p(wd), cout, cin, kh, kw, _p(alpha), _p(ws), _p(wm), _p(wf), _p(wtt),
                                   _p(wf8), _p(gs), _p(igs), fmt, _stream()), "weight_pack")
    torch.cuda.synchronize()
    a_ref = B.weight_alpha(wt.double()).float()
    torch.testing.assert_close(alpha.cpu(), a_ref, rtol=2e-6, atol=0)
    assert torch.equal(_as_u32(ws), B.pack_weight_bits(wt))
    assert torch.equal(_as_u32(wm), B.pack_flat_mask(wt))
    sg = B.sign_pm1(wt).reshape(cout, cin, T)
    assert torch.equal(wf.float().cpu(), sg.permute(0, 2, 1))
    assert torch.equal(wf8.view(torch.float8_e4m3fn).float().cpu(), sg.permute(0, 2, 1))
    live = (alpha.cpu() > 0).float().view(cout, 1, 1)
    exp_wt = (sg * live).flip(2).permute(1, 2, 0)          # [cin, T(flipped), cout]
    assert torch.equal(wtt.float().cpu(), exp_wt)
    exp_gs = torch.where(alpha.cpu() > 0, alpha.cpu(), torch.ones(cout))
    assert torch.equal(gs.cpu(), exp_gs)
    torch.testing.assert_close(igs.cpu(), 1.0 / exp_gs, rtol=1e-6, atol=0)


CONV_SHAPES = [  # n, cin, h, w, cout, k, stride, pad
    (2, 64, 8, 8, 64, 3, 1, 1), (1, 16, 9, 7, 16, 3, 1, 1), (2, 32, 8, 8, 64, 3, 2, 1),
    (1, 128, 5, 5, 32, 1, 2, 0), (2, 40, 6, 7, 8, 3, 2, 1), (2, 33, 5, 4, 5, 3, 1, 0),
    (1, 8, 7, 7, 24, 5, 1, 2), (1, 256, 4, 4, 128, 3, 1, 1), (3, 3, 6, 6, 7, 3, 1, 1),
    (1, 64, 1, 1, 64, 3, 1, 1), (1, 512, 3, 3, 64, 3, 1, 1),
]


def _run_fwd(x, wt, stride, pad, impl="xnor"):
    from bdbnn_b200.functional import binconv2d
    return binconv2d(x.cuda().contiguous(memory_format=torch.channels_last), wt.cuda(), stride, pad, impl)


@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_binconv_fwd_xnor_integer_exact_and_scaled(shape):
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(3 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g)
    x.view(-1)[0] = 0.0
    # (a) |W| == 0.5 everywhere -> alpha == 0.5 exactly -> y = 0.5 * integer, bit-exact comparison
    wt = B.sign_pm1(torch.randn(cout, cin, k, k, generator=g)) * 0.5
    y = _run_fwd(x, wt, stride, pad)
    ref_int = B.binconv_int(x, wt, stride, pad)
    assert torch.equal(y.cpu(), ref_int * 0.5)
    # (b) generic weights: fp32 result of alpha * int, compared with the fp64 oracle
    wt = torch.randn(cout, cin, k, k, generator=g) * 0.2
    y = _run_fwd(x, wt, stride, pad)
    ref = B.binconv_forward(x.double(), wt.double(), stride, pad).float()
    torch.testing.assert_close(y.cpu(), ref, rtol=3e-6, atol=0)
    assert y.is_contiguous(memory_format=torch.channels_last) or y.numel() == y.shape[1]


@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_binconv_backward_generic_vs_oracle(shape):
    from bdbnn_b200.functional import binconv2d
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(5 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g) * 1.2
    wt = torch.randn(cout, cin, k, k, generator=g) * 0.8          # some |W| > 1 -> weight STE mask active
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = wt.cuda().requires_grad_(True)
    y = binconv2d(xd, wd, stride, pad, "xnor")
    gy = torch.randn(y.shape, generator=g)
    y.backward(gy.cuda())
    gx_ref, gw_ref = B.binconv_backward(x.double(), wt.double(), gy.double(), stride, pad)
    # fp32 accumulation over K = cout*k*k (dgrad) / n*ho*wo (wgrad) terms: tolerance relative to max |.|
    for got, ref in ((xd.grad.cpu(), gx_ref), (wd.grad.cpu(), gw_ref)):
        scale = ref.abs().max().item() + 1e-30
        assert (got.double() - ref).abs().max().item() <= 2e-5 * scale
    assert (xd.grad.cpu()[x.abs() > 1] == 0).all()
    assert (wd.grad.cpu()[wt.abs() > 1] == 0).all()


def test_module_matches_oracle_module_nchw_input():
    """NCHW-contiguous input (not channels_last) goes through the layout conversion transparently."""
    from bdbnn_b200 import HardBinaryConv
    torch.manual_seed(0)
    conv = HardBinaryConv(32, 48, 3, 2, 1).cuda()
    ref = B.RefBinarizeConv2d(32, 48, 3, 2, 1)
    ref.load_state_dict(conv.state_dict())
    x = torch.randn(2, 32, 11, 9)
    xd = x.cuda().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    y, yr = conv(xd), ref(xr)
    torch.testing.assert_close(y.cpu(), yr, rtol=1e-5, atol=1e-6)
    gy = torch.randn_like(yr)
    y.backward(gy.cuda())
    yr.backward(gy)
    torch.testing.assert_close(xd.grad.cpu(), xr.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(conv.weight.grad.cpu(), ref.weight.grad, rtol=1e-4, atol=1e-4)
    with torch.no_grad():
        assert conv(xd).shape == (2, 48, 6, 5)


def test_forward_sign_flip_symmetry_at_baseline_size():
    """Size-independent property at the BASELINE.json config-2 layer shape (ResNet-18 layer1, N=256):
    y(-x) == -y(x) exactly when x has no zeros; and per-output |y|/alpha has the parity of K."""
    from bdbnn_b200.functional import binconv2d
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(256, 64, 56, 56, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    x[x == 0] = 1.0
    w = B.sign_pm1(torch.randn(64, 64, 3, 3, device="cuda", generator=g)) * 0.25
    y1 = binconv2d(x, w, 1, 1, "xnor")
    y2 = binconv2d(-x, w, 1, 1, "xnor")
    assert torch.equal(y1, -y2)
    inner = (y1[:, :, 1:-1, 1:-1] / 0.25)
    assert torch.equal(inner, inner.round())
    assert ((inner.to(torch.int64) - 576) % 2 == 0).all()        # K = 576 taps*channels: same parity
    assert inner.abs().max() <= 576


# ---- losses ---------------------------------------------------------------------------------------
def _golden(name):
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", name), weights_only=False)


def test_kurtosis_dropin_matches_reference_golden():
    from bdbnn_b200 import KurtosisWeight
    for case in _golden("kurtosis_cases.pt"):
        w = case["w"].cuda().requires_grad_(True)
        obj = KurtosisWeight(w, "w", kurtosis_target=case["target"], k_mode=case["mode"])
        assert obj.fn_regularization() is None
        obj.kurtosis_loss.backward()
        # the reference computes in fp32 (its own round-off ~1e-6 rel); we accumulate in fp64
        torch.testing.assert_close(obj.kurtosis.cpu(), case["kurtosis"], rtol=2e-5, atol=0)
        torch.testing.assert_close(obj.kurtosis_loss.detach().cpu(), case["loss"], rtol=2e-4, atol=1e-7)
        scale = case["grad"].abs().max().item()
        assert (w.grad.cpu() - case["grad"]).abs().max().item() <= 3e-4 * scale
        # against the fp64 oracle the kernel is tighter
        k64, l64 = Lr.kurtosis_ref(case["w"].double(), case["target"])
        g64 = Lr.kurtosis_grad_ref(case["w"].double(), case["target"])
        torch.testing.assert_close(obj.kurtosis.cpu().double(), k64, rtol=1e-6, atol=0)
        assert (w.grad.cpu().double() - g64).abs().max().item() <= 5e-6 * g64.abs().max().item()
        assert obj.KLDiv_loss == 0


def test_kurtosis_multi_19_layers_and_modes():
    from bdbnn_b200 import kurtosis_regularization
    g = torch.Generator().manual_seed(2)
    shapes = [(64, 64, 3, 3)] * 4 + [(128, 64, 3, 3), (128, 128, 3, 3), (128, 64, 1, 1)] + [(256, 256, 3, 3)] * 2 \
        + [(33,), (7, 5, 3, 3)] + [(512, 512, 3, 3)] + [(16, 16, 3, 3)] * 7
    assert len(shapes) == 19
    ws = [(torch.randn(s, generator=g) * 0.05 + 0.01 * i) for i, s in enumerate(shapes)]
    targets = [1.8, 1.4, 1.4, 1.4, 1.4, 1.2, 1.4, 1.2, 1.2, 1.4, 1.4, 1.4, 1.2, 1.2, 1.2, 1.2, 1.4, 1, 1]
    for mode in ("avg", "sum", "max"):
        wd = [w.cuda().requires_grad_(True) for w in ws]
        reg, losses, kurt = kurtosis_regularization(wd, targets, mode, len(wd), 0.7)
        reg.backward()
        wr = [w.double().requires_grad_(True) for w in ws]
        ref_l = [Lr.kurtosis_ref(w, t)[1] for w, t in zip(wr, targets)]
        ref = Lr.aggregate_kurtosis(ref_l, mode, len(wr), 0.7)
        ref.backward()
        torch.testing.assert_close(reg.detach().cpu().double(), ref.detach(), rtol=1e-5, atol=0)
        for a, b in zip(wd, wr):
            scale = b.grad.abs().max().item()
            if scale == 0:
                assert a.grad.abs().max().item() == 0
            else:
                assert (a.grad.cpu().double() - b.grad).abs().max().item() <= 1e-5 * scale


def test_kd_logits_matches_reference_golden():
    from bdbnn_b200 import DistributionLoss
    crit = DistributionLoss().cuda()
    for case in _golden("kd_logits_cases.pt"):
        s = case["s"].cuda().requires_grad_(True)
        loss = crit(s, case["t"].cuda())
        (loss * 0.9).backward()                       # alpha scaling as at train.py:612
        torch.testing.assert_close(loss.detach().cpu(), case["loss"], rtol=3e-6, atol=1e-6)
        torch.testing.assert_close(s.grad.cpu(), case["grad"] * 0.9, rtol=2e-5, atol=1e-8)


def test_kd_layer_matches_reference_golden():
    from bdbnn_b200 import DistributionLoss_layer
    from helpers import tiny_net as _tiny
    for case in _golden("kd_layer_cases.pt"):
        stud, teach = _tiny(case["wrapped"]), _tiny(case["wrapped"])
        stud.load_state_dict(case["stud_state"])
        teach.load_state_dict(case["teach_state"])
        stud, teach = stud.cuda(), teach.cuda()
        loss = DistributionLoss_layer()(None, None, stud, teach, 4)
        (loss * 200.0).backward()                     # beta scaling as at train.py:611
        torch.testing.assert_close(loss.detach().cpu(), case["loss"], rtol=2e-6, atol=1e-7)
        for n, p in stud.named_parameters():
            gref = case["grads"][n]
            if gref is None:
                assert p.grad is None
            else:
                torch.testing.assert_close(p.grad.cpu(), gref * 200.0, rtol=2e-6, atol=1e-9)


@pytest.mark.parametrize("geom", [(2, 64, 16, 16, 3, 2, 1), (1, 8, 7, 9, 3, 2, 1), (2, 4, 6, 6, 2, 2, 0),
                                  (1, 16, 9, 9, 3, 1, 1), (1, 64, 112, 112, 3, 2, 1)])
def test_maxpool_nhwc_matches_torch(geom):
    from bdbnn_b200.functional import max_pool2d_nhwc
    import torch.nn.functional as F
    n, c, h, w, k, s, p = geom
    g = torch.Generator().manual_seed(sum(geom))
    x = torch.randn(n, c, h, w, generator=g)
    x[0, 0, 0, 0] = float("nan")
    x[0, 1, :, :] = 0.5                                   # ties everywhere in this plane
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    y = max_pool2d_nhwc(xd, k, s, p)
    yr = F.max_pool2d(xr, k, s, p)
    assert torch.equal(torch.nan_to_num(y.cpu(), nan=7.0), torch.nan_to_num(yr.detach(), nan=7.0))
    gy = torch.randn(yr.shape, generator=g)
    y.backward(gy.cuda())
    yr.backward(gy)
    # tie plane: the gradient mass per window must match even if the tie-break differs; elsewhere exact
    gd, gr = xd.grad.cpu(), xr.grad
    sel = torch.ones(c, dtype=torch.bool); sel[1] = False
    gd0, gr0 = torch.nan_to_num(gd[:, sel]), torch.nan_to_num(gr[:, sel])
    torch.testing.assert_close(gd0, gr0, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(gd[:, 1].sum(), gr[:, 1].sum(), rtol=1e-5, atol=1e-5)


def test_bits_to_fp8():
    _lib, L, _p, _stream, _ = _env()
    g = torch.Generator().manual_seed(9)
    x = torch.randn(3, 64, 5, 7, generator=g)
    bits = B.pack_bits_nhwc(x).to(torch.int32).cuda()          # low 32 bits
    out = torch.zeros((3, 5, 7, 64), dtype=torch.uint8, device="cuda")
    _lib.check(L.bdbnn_bits_to_fp8(_p(bits), 3 * 5 * 7, 64, _p(out), _stream()), "bits_to_fp8")
    assert torch.equal(out.view(torch.float8_e4m3fn).float().cpu(), B.sign_pm1(x).permute(0, 2, 3, 1))


@pytest.mark.parametrize("impl,shape,tol", [("xnor", (2, 16, 9, 8, 24, 3, 1, 1), 2e-5),
                                            ("xnor", (2, 32, 8, 8, 32, 3, 2, 1), 2e-5),
                                            ("tc", (4, 64, 8, 8, 64, 3, 1, 1), 1.5e-3)])
@pytest.mark.parametrize("kt", [(1.0, 1.0), (3.1623, 0.3162), (1.0, 9.4406)])
def test_ede_backward_vs_oracle(impl, shape, tol, kt):
    """EDE backward (train.py:409-415): forward unchanged, both STE indicators replaced by
    k*t*(1 - tanh(t*v)^2); k/t stay device tensors."""
    from bdbnn_b200.functional import binconv2d
    n, cin, h, w, cout, ks, stride, pad = shape
    g = torch.Generator().manual_seed(11 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g) * 1.2
    wt = torch.randn(cout, cin, ks, ks, generator=g) * 0.8
    k, t = torch.tensor([kt[0]]), torch.tensor([kt[1]])
    xd = _nhwc(x).requires_grad_(True)
    wd = wt.cuda().requires_grad_(True)
    y = binconv2d(xd, wd, stride, pad, impl, (k.cuda(), t.cuda()))
    y0 = binconv2d(xd.detach(), wd.detach(), stride, pad, impl)
    assert torch.equal(y.detach(), y0)                               # forward is not touched by EDE
    gy = torch.randn(y.shape, generator=g)
    y.backward(gy.cuda())
    gx_ref, gw_ref = B.binconv_backward_ede(x.double(), wt.double(), gy.double(), k.double(), t.double(), stride, pad)
    for got, ref in ((xd.grad.cpu(), gx_ref), (wd.grad.cpu(), gw_ref)):
        scale = ref.abs().max().item() + 1e-30
        assert (got.double() - ref).abs().max().item() <= tol * scale


def test_ede_module_cifar_follows_assigned_k_t():
    """HardBinaryConv_cifar switches to the EDE backward once the loop assigned .k/.t; the oracle
    module does the same; HardBinaryConv ignores the attributes."""
    from bdbnn_b200 import HardBinaryConv, HardBinaryConv_cifar
    from bdbnn_b200.step import apply_ede
    torch.manual_seed(3)
    x = torch.randn(2, 16, 10, 10) * 1.3
    for cls, reacts in ((HardBinaryConv_cifar, True), (HardBinaryConv, False)):
        conv = cls(16, 32, 3, 1, 1).cuda()
        ref = B.RefBinarizeConv2d(16, 32, 3, 1, 1)
        ref.load_state_dict(conv.state_dict())
        ref.supports_ede = reacts
        t, k = apply_ede(conv, 30, 120)
        ref.k, ref.t = k.cpu(), t.cpu()
        xd = _nhwc(x).requires_grad_(True)
        xr = x.clone().requires_grad_(True)
        y, yr = conv(xd), ref(xr)
        gy = torch.randn_like(yr)
        y.backward(gy.cuda())
        yr.backward(gy)
        torch.testing.assert_close(y.detach().cpu(), yr.detach(), rtol=1e-5, atol=1e-6)
        # 16/32-channel shapes run on the wgmma path: fp16s gradient operand -> 1.5e-3 of max|ref|
        for got, want in ((xd.grad.cpu(), xr.grad), (conv.weight.grad.cpu(), ref.weight.grad)):
            assert (got - want).abs().max().item() <= 1.5e-3 * want.abs().max().item()
